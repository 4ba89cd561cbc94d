/*
 * nvwn_b200.h -- handle-based C-ABI of the WaveNet inference engine.
 *
 * One entry point per public member of the reference's host class
 * nvWavenetInfer<T_weight,T_data,R,S,A> (nv_wavenet.cuh:220-640), so that the C++ facade
 * (include/nv_wavenet.hpp), the reference C-ABI (include/wavenet_infer.h) and any FFI
 * (ctypes, cgo, JNI ...) can drive the same engine.  Plain pointers and sizes only.
 *
 * Conventions
 *   - every function returns 0 on success, a cudaError_t (>0) or a negative NVWN_E* code on
 *     failure; nvwn_last_error() gives the message (thread-local).
 *   - every float* / int* data argument may be host or device memory (cudaMemcpyDefault),
 *     like the reference setters (nv_wavenet.cuh:285-308); data is copied before return.
 *   - matrices fp32 column-major M x K; embeddings [A][R]; Lh float[N][L][B][2R];
 *     selectors float[N][B]; yOut int[B][N]  (nv_wavenet.cuh:144, singleblock.cuh:232,245).
 *   - `stream` is a cudaStream_t passed as void* (NULL = default stream).
 */
#ifndef NVWN_B200_H
#define NVWN_B200_H

#ifdef __cplusplus
extern "C" {
#endif

typedef struct nvwn_engine nvwn_engine;

enum { NVWN_FP32 = 0, NVWN_FP16 = 1,          /* T_data=float (bit-exact to the reference CPU model) / T_data=half of the reference */
       NVWN_FP32_FAST = 2 };                  /* fp32 in the reference GPU kernels' arithmetic: FMA, two interleaved partial sums per dot
                                                 product (matrix_math.cuh:80-117), float libm tanh/exp -- agrees with the CPU model like the
                                                 reference's own kernels do (nv_wavenet_test.cu:273-298), about twice as fast */
enum { NVWN_EINVAL = -1, NVWN_EUNSUPPORTED = -2, NVWN_ENOMEM = -3 };
/* kernel selection; the reference's Implementation enum values 0..4 are accepted and map to AUTO */
enum { NVWN_KERNEL_AUTO = 0, NVWN_KERNEL_STREAM = 16, NVWN_KERNEL_TENSORCORE = 17, NVWN_KERNEL_LATENCY = 18 };

/* nvWavenetInfer::nvWavenetInfer (nv_wavenet.cuh:311) */
int nvwn_create(nvwn_engine** out, int dtype, int R, int S, int A, int num_layers, int max_dilation,
                int batch_size, int num_samples, int impl, int tanh_embed);
/* nvWavenetInfer::~nvWavenetInfer (nv_wavenet.cuh:362-395) */
int nvwn_destroy(nvwn_engine* e);
const char* nvwn_last_error(void);

/* nv_wavenet.cuh:396-415 */
int nvwn_set_embeddings(nvwn_engine* e, const float* embedPrev, const float* embedCur);
int nvwn_set_layer_weights(nvwn_engine* e, int layer, const float* Wprev, const float* Wcur, const float* Bh,
                           const float* Wres, const float* Bres, const float* Wskip, const float* Bskip);
int nvwn_set_out_weights(nvwn_engine* e, const float* Wzs, const float* Bzs, const float* Wza, const float* Bza);
/* nv_wavenet.cuh:417-422: resets the feedback history to 128/128, copies Lh and selectors */
int nvwn_set_inputs(nvwn_engine* e, const float* Lh, const float* selectors);
/* extension: selectors only / conditioning only (conditioning may be uploaded in chunks of whole samples) */
int nvwn_set_selectors(nvwn_engine* e, const float* selectors);
int nvwn_set_conditioning(nvwn_engine* e, const float* Lh, int first_sample, int num_samples, void* stream);
/* extension (SURVEY.md 8f next-1): selectors drawn ON THE DEVICE, counter-based and stateless -- selector[i], i = sample *
 * batch_size + b, is the first output of Philox-4x32-10 with counter (i, 0) and key `seed`, as (x >> 8) * 2^-24 in [0, 1)
 * (the reference draws them on the host with libc rand(), pytorch/wavenet_infer.cu:92-93).  Asynchronous on `stream`. */
int nvwn_set_selectors_random(nvwn_engine* e, unsigned long long seed, void* stream);
/* Streaming (see nvwn_run_stream): the selectors of absolute samples [first_sample, first_sample + num_samples), num_samples <=
 * num_samples of the engine: selector (t, b) from counter t * batch_size + b, stored at position t mod num_samples.  For t < N
 * these are the values nvwn_set_selectors_random writes; they do not depend on the engine's num_samples. */
int nvwn_set_selectors_random_stream(nvwn_engine* e, unsigned long long seed, long long first_sample, int num_samples, void* stream);
/* host helper (needs no GPU): the selectors exactly as the reference wrapper draws them -- Matrix(batch, samples).randomize(0.5, 1.0)
 * on the caller's libc rand() stream (pytorch/wavenet_infer.cu:92-93, matrix.cpp:38-56) -- into selectors[sample * batch_size + b]. */
int nvwn_libc_selectors(float* selectors, int batch_size, int sample_count);
/* Conditioning producer on the device (SURVEY.md 8f next-2).  Replaces, for inference, WaveNet.get_cond_input
 * (pytorch/wavenet.py:190-202: ConvTranspose1d(C, C, window, stride) upsampling trimmed by window - stride, then the
 * 1x1 cond_layers convolution C -> L*2R) and the permutes to [N][L][B][2R] (pytorch/nv_wavenet.py:48-49,181):
 *   features [B][C][T] (mel frames), upsample_weight [C][C][window] (torch ConvTranspose1d layout), upsample_bias [C],
 *   cond_weight [L*2R][C] (Conv1d weight, kernel size 1), cond_bias [L*2R]; all fp32, host or device memory.
 * Produces conditioning for samples [first_sample, first_sample + T*stride) in chunks, directly in the engine's
 * conditioning store -- the [N][L][B][2R] fp32 tensor never exists.  Returns after the work has completed. */
int nvwn_set_conditioning_from_features(nvwn_engine* e, const float* features, int n_cond_channels, int num_frames,
                                        const float* upsample_weight, const float* upsample_bias, int window, int stride,
                                        const float* cond_weight, const float* cond_bias, int first_sample, void* stream);
/* The same in two steps, for producers that run concurrently with generation: _load copies the features and the two layers' weights
 * into engine-owned device memory (returns when the sources may be released); _run fills conditioning for samples
 * [sample_begin, sample_begin + sample_count) of the loaded sequence, stored from engine sample first_sample + sample_begin,
 * asynchronously on `stream` (order it before the nvwn_run_partial that consumes those samples with an event; successive _run
 * calls must be on one stream or ordered by the caller: they share scratch). */
int nvwn_cond_producer_load(nvwn_engine* e, const float* features, int n_cond_channels, int num_frames,
                            const float* upsample_weight, const float* upsample_bias, int window, int stride,
                            const float* cond_weight, const float* cond_bias, void* stream);
int nvwn_cond_producer_run(nvwn_engine* e, int first_sample, int sample_begin, int sample_count, void* stream);
/* Streaming (see nvwn_run_stream): samples [sample_begin, sample_begin + sample_count) of the loaded sequence, sample s stored at
 * position s mod num_samples; sample_count <= num_samples.  Asynchronous on `stream` like nvwn_cond_producer_run. */
int nvwn_cond_producer_run_stream(nvwn_engine* e, long long sample_begin, int sample_count, void* stream);
/* Live vocoding: mel frames that arrive over time, a few at a time, into a bounded ring on the device, and conditioning produced
 * for each sample as soon as its frames are in.  Sample n reads frames ceil((n - window + 1) / stride) .. floor(n / stride) only,
 * so its conditioning is final, bit for bit, once frame floor(n / stride) has been pushed: the same bits nvwn_cond_producer_load
 * of the finished frames gives it.
 *
 * _open_live starts a live sequence of 0 frames for the B rows on the whole-batch producer, with a ring of ring_frames frames per
 * row; ring_frames < ceil(window / stride) + 1 is NVWN_EINVAL.  The network as for nvwn_cond_producer_load; returns when the
 * sources may be released.  It replaces a loaded sequence, and nvwn_cond_producer_load ends a live one.
 * _push appends features [B][n_cond_channels][num_frames] (host or device memory) as frames [T, T + num_frames) of the sequence,
 * T the frames pushed so far.  A host array may be reused on return; device frames are copied in order on `stream`.  A push that
 * would overwrite a frame a sample not produced yet reads (one at or past the end of the furthest nvwn_cond_producer_run_stream of
 * this sequence) is NVWN_EINVAL and changes nothing; num_frames = 0 does nothing.  A sequence holds at most INT_MAX samples.
 * nvwn_cond_producer_run_stream on a live sequence takes samples below T * stride whose frames are all still in the ring (else
 * NVWN_EINVAL, naming the first missing frame); nvwn_cond_producer_run refuses a live sequence.  Issue pushes and productions on
 * one stream, or order them: a push writes ring columns that earlier productions read. */
int nvwn_cond_producer_open_live(nvwn_engine* e, int n_cond_channels, const float* upsample_weight, const float* upsample_bias, int window,
                                 int stride, const float* cond_weight, const float* cond_bias, int ring_frames, void* stream);
int nvwn_cond_producer_push(nvwn_engine* e, const float* features, int num_frames, void* stream);
/* The same arithmetic on the host (needs no GPU; test / reference use): Lh [T*stride][L][B][2R], host pointers. */
int nvwn_cond_from_features_host(float* Lh, const float* features, int batch_size, int n_cond_channels, int num_frames,
                                 const float* upsample_weight, const float* upsample_bias, int window, int stride,
                                 const float* cond_weight, const float* cond_bias, int num_layers, int R);
int nvwn_reset_history(nvwn_engine* e);
/* extension (teacher forcing): forced[b*num_samples + t] is fed back instead of the sampled index;
 * NULL switches it off.  Copied. */
int nvwn_set_forced(nvwn_engine* e, const int* forced);
/* extension: replicate rank `root`'s packed weights to every rank's engine is done by the caller
 * (NCCL broadcast of the blob below); these expose the packed device blob. */
int nvwn_weight_blob(nvwn_engine* e, void** dev_ptr, unsigned long long* bytes);
/* must be called after the blob was overwritten (e.g. by an NCCL broadcast) */
int nvwn_weights_updated(nvwn_engine* e);

/* nv_wavenet.cuh:499-639.  run_partial generates samples [init_sample, init_sample+count) of a
 * num_samples-long utterance batch; yOut (optional, host or device) receives the whole int[B][N]. */
int nvwn_run_partial(nvwn_engine* e, int init_sample, int count, int num_samples, int batch_size,
                     int* yOut, int dump_activations, void* stream);
int nvwn_run(nvwn_engine* e, int num_samples, int batch_size, int* yOut, int dump_activations, void* stream);
/* Streaming generation: utterances of any length through an engine of num_samples = N.  The N-sample buffers are rings: absolute
 * sample t of the utterance batch uses position t mod N of the conditioning, the selectors, the forced indices and yOut (row stride
 * N), while the history goes by t itself.  So the result is bit-identical to one engine that holds the whole length.  Generates
 * absolute samples [first_sample, first_sample + count), count <= N, in at most two launches (split at the wrap; dumps come from the
 * last).  first_sample must be the engine's next sample: 0 after nvwn_reset_history / nvwn_set_inputs, else the end of the last
 * generation (nvwn_run_partial / nvwn_run included); any other value is NVWN_EINVAL.  batch_size as for nvwn_run_partial.
 * Fill the positions of a range (conditioning, selectors, forced indices) before the call, and read them (nvwn_get_yout,
 * nvwn_get_audio) before a later call overwrites them. */
int nvwn_run_stream(nvwn_engine* e, long long first_sample, int count, int batch_size, int dump_activations, void* stream);
/* Continuous batching: the B rows of a streaming engine are slots, each serving one utterance after another.  Between launches a
 * slot's whole state is its row of the history ring and its two fed-back indices, so a new utterance starts in a slot while the
 * others keep going.  slots / seeds are host arrays of n distinct slots in [0, B), 1 <= n <= B, copied before return (the caller
 * may reuse them at once, pinned or not).  The rows these calls write (history, conditioning, selectors) are laid out for runs of
 * the whole batch: after any of them, and until nvwn_reset_history, nvwn_run_stream / nvwn_run_partial with batch_size != B is
 * NVWN_EINVAL.  The calls share the engine's slot scratch: issue them on one stream, or order them.
 *
 * Start a new utterance in each of slots[0..n) at the engine's next sample t0 (the first_sample the next nvwn_run_stream takes):
 * that row's history is cleared and its fed-back indices set to 128, exactly as at a fresh start; the other rows are not touched.
 * seeds (NULL = all 0) key the slot's selectors for nvwn_set_selectors_random_slots.  Stream-ordered on `stream`: issue it
 * after the launch that ends at t0.  nvwn_reset_history sets every slot's start to 0 and its seed to 0. */
int nvwn_restart_slots(nvwn_engine* e, const int* slots, int n, const unsigned long long* seeds, void* stream);
/* Lh [num_samples][L][n][2R] fp32 (host or device): conditioning of absolute samples [first_sample, +num_samples) for rows
 * slots[0..n) only, sample t at position t mod N; num_samples <= N (split at the wrap inside).  A host Lh is staged and the call
 * returns when it may be released; a device Lh is converted asynchronously on `stream`. */
int nvwn_set_conditioning_slots(nvwn_engine* e, const float* Lh, const int* slots, int n, long long first_sample, int num_samples, void* stream);
/* selectors of absolute samples [first_sample, +num_samples), num_samples <= N, for every slot from its (seed, origin): slot b at
 * sample t gets the Philox draw of counter t - origin[b] under key seed[b] (mapped as nvwn_set_selectors_random), which is what
 * nvwn_set_selectors_random_stream(seed[b], ...) gives a one-utterance engine at sample t - origin[b]: an utterance's selectors do
 * not depend on its slot, its start or the batch it shares.  Asynchronous on `stream`. */
int nvwn_set_selectors_random_slots(nvwn_engine* e, long long first_sample, int num_samples, void* stream);
/* Per-slot conditioning producer: each slot's conditioning made on the device from its own utterance's mel frames, straight into
 * that slot's rows of the store (the arithmetic of nvwn_set_conditioning_from_features, utterance by utterance).  The three calls
 * have their own weights and scratch, apart from nvwn_cond_producer_load / _run, and use neither the slot scratch of the calls
 * above nor the restart state: they may run on a side stream while the generating stream restarts slots and generates, ordered
 * only by events (issue the three on one stream: they share scratch).  _set_slots and _run_slots count as per-slot calls for the
 * whole-batch rule above.
 *
 * The conditioning network, as for nvwn_set_conditioning_from_features (host or device memory).  Returns when the sources may be
 * released.  Forgets the frames attached to every slot. */
int nvwn_cond_producer_set_weights(nvwn_engine* e, int n_cond_channels, const float* upsample_weight, const float* upsample_bias, int window,
                                   int stride, const float* cond_weight, const float* cond_bias, void* stream);
/* Attaches utterance i, frames features[i] [n_cond_channels][num_frames[i]] (num_frames[i] >= 1), to slot slots[i]; its sample 0 is
 * absolute sample starts[i] >= 0 and it has num_frames[i] * stride samples.  The frames are copied into engine memory: host frames
 * are staged and may be released on return, device frames are copied in stream order on `stream`.  The host arrays (slots,
 * features, num_frames, starts) may be reused on return, pinned or not.  nvwn_reset_history forgets every attached utterance. */
int nvwn_cond_producer_set_slots(nvwn_engine* e, const int* slots, int n, const float* const* features, const int* num_frames,
                                 const long long* starts, void* stream);
/* Conditioning of absolute samples [first_sample, first_sample + num_samples), num_samples <= N, for rows slots[0..n) only, sample t
 * at position t mod N: slot s gets sample t - start of its utterance, and 0 at or past that utterance's end.  Every listed slot needs
 * an attached utterance with start <= first_sample.  Asynchronous on `stream`; other rows are not touched. */
int nvwn_cond_producer_run_slots(nvwn_engine* e, const int* slots, int n, long long first_sample, int num_samples, void* stream);
/* Live frames for single slots: each slot's utterance gets its mel frames as they arrive, into a ring of its own, as the whole-batch
 * live sequence of nvwn_cond_producer_open_live does for a batch that moves in lockstep.
 *
 * _open_live_slots switches the per-slot producer (after nvwn_cond_producer_set_weights) to rings of ring_frames >= ceil(window /
 * stride) + 1 frames per slot and forgets every attached utterance.  Until nvwn_cond_producer_set_weights or nvwn_reset_history
 * leaves this live mode, _set_slots is NVWN_EINVAL. */
int nvwn_cond_producer_open_live_slots(nvwn_engine* e, int ring_frames, void* stream);
/* Slot slots[i] takes a live utterance whose sample 0 is absolute sample starts[i] (negative for a resumed utterance further along than
 * the engine), with its frames [first_frames[i], first_frames[i] + num_frames[i]) given as features[i] [n_cond_channels][num_frames[i]],
 * num_frames[i] <= ring_frames; the frames before first_frames[i] count as pushed but have left the ring.  A fresh utterance passes
 * first_frames 0 and num_frames 0, and may pass NULL features.  Host frames may be reused on return; device frames are copied in
 * order on `stream`. */
int nvwn_cond_producer_attach_live(nvwn_engine* e, const int* slots, int n, const long long* starts, const int* first_frames,
                                   const float* const* features, const int* num_frames, void* stream);
/* Appends features[i] [n_cond_channels][num_frames[i]] to slot slots[i]'s live utterance.  Refused with NVWN_EINVAL, changing nothing,
 * when a push would overwrite a frame that a sample of that slot not produced yet reads (as nvwn_cond_producer_push), or a slot has no
 * live utterance.  Host frames may be reused on return.
 * nvwn_cond_producer_run_slots produces a live slot from its ring: its end is T * stride for the T frames pushed so far, samples past
 * it are 0, and a range whose first sample reads a frame no longer in the ring is NVWN_EINVAL. */
int nvwn_cond_producer_push_slots(nvwn_engine* e, const int* slots, int n, const float* const* features, const int* num_frames, void* stream);
/* nv_wavenet.cuh:439-444: 2-D copy of yOut[b][offset .. offset+size) for every b */
int nvwn_get_yout(nvwn_engine* e, int* yOut, int offset, int size, void* stream);
/* Output side (SURVEY.md 8f next-3): replaces the host post-processing of pytorch/nv_wavenet_inference.py:55-60 --
 * utils.mu_law_decode_numpy (pytorch/utils.py:62-70) with mu_quantization = A, then MAX_WAV_VALUE * audio and
 * astype('int16') -- on the device, straight from the engine's yOut: audio[b][j] for j in [0, size) decodes
 * yOut[b][offset + j].  audio_f32 (in [-1, 1]) and / or audio_i16 may be NULL; each is [B][size], host or device memory
 * (device destinations are filled asynchronously on `stream`).  Table-driven, the table computed on the host in double
 * exactly as numpy does, so values equal the reference's.  saturate = 0 keeps the reference's cast (code A-1 decodes to
 * +1.0 -> 32768 -> wraps to -32768), saturate = 1 clamps to 32767. */
int nvwn_get_audio(nvwn_engine* e, float* audio_f32, short* audio_i16, int offset, int size, int saturate, void* stream);
/* The decode table itself (host only, needs no GPU): entry x = decoded value of code x for mu_quantization = A; any of
 * the three outputs (A entries each) may be NULL. */
int nvwn_mulaw_table(int A, float* f32, short* i16_wrap, short* i16_saturate);

/* Teacher-forced scoring.  logp[b*num_samples + t] = log softmax(Za_t)[audio[b*num_samples + t]], where Za_t are the logits
 * generation would compute at step t from silence with audio[b][0..t) fed back (teacher forcing): the embedding input of step t
 * is (audio[t-2], audio[t-1]) with audio[-1] = audio[-2] = 128, x_l[t-d] = 0 for t < d, and step t uses the conditioning Lh[t]
 * in the engine's store (set_inputs, set_conditioning or the conditioning producer).  All steps are computed at once, over
 * the first batch_size utterances of the store (batch_size <= B, num_samples <= N).  logits (NULL, or [batch_size][num_samples][A])
 * receives the fp32 logits.  audio, logp and logits may each be host or device memory; the call returns after completion if
 * any destination is on the host, device destinations are filled asynchronously on `stream`.  The generation state (history,
 * yOut, selectors, forced indices, dumps, launch info) is left untouched.  Each output (b, t) depends only on audio[b][0..t],
 * the conditioning and the weights, bit for bit.  NVWN_FP16 engines with A = 256 only (else NVWN_EUNSUPPORTED); an audio value
 * outside [0, A) is NVWN_EINVAL and the message names the first offending (b, t).  Ends the scoring stream below. */
int nvwn_score(nvwn_engine* e, const int* audio, int num_samples, int batch_size,
               float* logp, float* logits, void* stream);
/* Streaming scoring: utterances of any length through an engine of num_samples = N, as nvwn_run_stream does for generation.
 * Scores absolute samples [first_sample, first_sample + count), 1 <= count <= N; audio and logp are [batch_size][count] and
 * logits (NULL, or [batch_size][count][A]) covers them too.  Sample t uses the conditioning at store position t mod N: fill a range's
 * positions before the call.  first_sample = 0 starts a scoring stream from silence; any other first_sample must continue it (the
 * end of the last call of the stream, with the same batch_size), else NVWN_EINVAL.  Between calls the engine keeps each layer's last
 * d_l inputs and the last two codes, so the results equal nvwn_score of one engine that holds the whole length, bit for bit.
 * nvwn_score and every weight change (the weight setters, nvwn_weights_updated) end the stream; generation calls leave it alone, and
 * it leaves the generation state alone.  A call that fails its checks (bad audio included) leaves the stream as it was.  Memory
 * kinds, completion, the audio check (the message names t as an absolute sample) and the engine kinds as for nvwn_score; the
 * calls share scratch with nvwn_score: issue them on one stream, or order them. */
int nvwn_score_stream(nvwn_engine* e, const int* audio, long long first_sample, int count, int batch_size,
                      float* logp, float* logits, void* stream);
/* Packed scoring: a queue of utterances scored end to end in the rows of one scoring stream (sequence packing).  Arguments and
 * results are those of nvwn_score_stream, plus starts [batch_size][count] (host or device memory): a nonzero starts[b][i] begins a
 * new utterance in row b at absolute sample first_sample + i.  Its codes of steps -1 and -2 are 128 and every layer's x_l[t - d]
 * reads 0 for t - d before that sample, so its results from that sample on are the bits nvwn_score gives that utterance alone, on
 * conditioning put at the same store positions.  first_sample = 0 opens a packed stream, and every row starts at sample 0 whatever
 * starts[b][0] says.  Between calls the engine keeps, besides the fronts and codes, each row's local time (samples since its
 * utterance began).  A stream is packed or not from its first call: continuing a packed stream with nvwn_score_stream, or one that
 * is not with this call, is NVWN_EINVAL; nvwn_prime_from_score and nvwn_prime_slots_from_score refuse a packed stream with
 * NVWN_EUNSUPPORTED (a row's fronts may hold an earlier utterance's inputs).  starts NULL is NVWN_EINVAL.  Every other rule --
 * continuation, ending, refused calls leaving the stream as it was, memory kinds, completion, engine kinds -- is nvwn_score_stream's. */
int nvwn_score_stream_packed(nvwn_engine* e, const int* audio, const unsigned char* starts, long long first_sample, int count,
                             int batch_size, float* logp, float* logits, void* stream);
/* Prompted generation: continue given audio.  Score the prompt, samples [0, P), with nvwn_score_stream (any windows), then this call
 * moves the open scoring stream's state into generation: for its batch_size Bs utterances, each layer's last d_l inputs go into the
 * history ring and the last two codes become the fed-back indices, and the engine's next sample becomes P.  Then
 * nvwn_run_stream(e, P, count, Bs, ...) generates the continuation; with nvwn_set_selectors_random_stream it draws at sample t what
 * any engine draws at t.  The scoring stream stays open and unchanged; nothing else changes (selectors, conditioning, forced indices,
 * per-slot state, dumps, launch info).  Stream-ordered on `stream`: issue it on the scoring calls' stream, or order them.
 * Needs an open scoring stream with P >= 1 (nvwn_score and weight changes end one), else NVWN_EINVAL; NVWN_FP16 engines only (else
 * NVWN_EUNSUPPORTED).  The tensor-core path, and any engine after a per-slot call, need Bs = B.  After a prime, and until
 * nvwn_reset_history, runs need batch_size = Bs (NVWN_EINVAL otherwise).  A refused call changes nothing.
 * Numerics: the primed history holds the scorer's fp16 layer inputs, whose GEMMs sum in another order than any generation kernel's,
 * so the continuation is not bit-identical to forced generation of the prompt.  It is bit-identical whatever the windows of the
 * scoring and generation calls, the primed history is the same on every engine kind, and it is within the fp16 contract of the
 * fp32 model at that history. */
int nvwn_prime_from_score(nvwn_engine* e, void* stream);
/* Prompted continuous batching: prime single slots of a running engine.  With an open scoring stream of batch_size Bs and next sample
 * P >= 1, and the engine's next sample t0: for each i, slot slots[i] starts an utterance whose samples [0, P) are scoring row rows[i],
 * its local time tau at engine time t0 - P + tau, so that generation from t0 continues it at tau = P.  The slots' history rows are
 * cleared, each layer's last d_l inputs of their rows go into them, the rows' last two codes become the fed-back indices, and the
 * slots' selector origin becomes t0 - P and their key seeds[i] (seeds NULL: 0): the same effect on those slots as nvwn_restart_slots
 * at t0 - P followed by a prime, so nvwn_set_selectors_random_slots draws counter tau, what an engine of that utterance alone draws.
 * A per-slot call (whole-batch runs until nvwn_reset_history).  The scoring stream stays open and unchanged, so rows of longer prompts
 * can be scored on and primed later; next_t does not move; no other slot changes.  Stream-ordered on `stream`.
 * The first such call since nvwn_reset_history at t0 < maxDil zeroes the history entries of the times [t0 - maxDil - 1, 0) in every
 * slot, and from then until nvwn_reset_history every launch reads the history at every step (the rows that started at sample 0 read
 * zeros where they staged zeros: the same bits, DESIGN.md §6).
 * Refused with NVWN_EINVAL, changing nothing: NULL rows or slots, no open scoring stream, rows outside [0, Bs) or given twice, a bad
 * slot list (1 <= n <= B, distinct slots in [0, B)).  NVWN_FP16 engines only (else NVWN_EUNSUPPORTED).  Numerics as
 * nvwn_prime_from_score. */
int nvwn_prime_slots_from_score(nvwn_engine* e, const int* rows, const int* slots, int n, const unsigned long long* seeds, void* stream);
/* Slot states: park a slot's utterance and resume it later, in any slot of any engine of the same dtype, R, L and maxDil.  Between
 * launches a slot's whole state is its history row, its two fed-back indices and its selector origin and seed, and an utterance's
 * samples do not depend on its slot, its start or its neighbours; so a saved and loaded utterance goes on with the bits it would
 * have had without the pause (DESIGN.md §6).  A state is a blob of nvwn_slot_state_bytes bytes, the same for every kernel family
 * and any B or N:
 *   - this 64-byte header, with position = the samples the utterance has generated or been primed with;
 *   - then for each layer l in order the layer inputs x_l of its times [position - d_l, position) as [d_l][R], in the ring's
 *     element type (fp16 on NVWN_FP16 engines, fp32 otherwise, so fp32 engines resume bit-exact); d_l = 1, 2, 4, ... doubling
 *     per layer and back to 1 past maxDil.  Times before 0 hold zeros. */
typedef struct {
    unsigned int tag;                   /* NVWN_SLOT_STATE_TAG */
    int dtype, R, L, max_dilation;
    int y_prev, y_cur;                  /* the fed-back indices: the codes of the two samples before `position` */
    int reserved0;
    long long position;
    unsigned long long seed;            /* the selector key (nvwn_restart_slots) */
    unsigned long long reserved[2];     /* zero */
} nvwn_slot_state_header;
enum { NVWN_SLOT_STATE_TAG = 0x3153564E };     /* "NVS1" */
int nvwn_slot_state_bytes(nvwn_engine* e, unsigned long long* bytes);
/* Writes the states of slots slots[0..n) at the engine's next sample to states + i * nvwn_slot_state_bytes, host or device memory
 * (16-byte aligned).  The engine does not change.  Device states are written asynchronously on `stream`; host states are complete
 * on return.  The slots' history rows are read at the engine's batch stride, where the per-slot calls and every run of the whole
 * batch keep them.  A bad slot list is NVWN_EINVAL. */
int nvwn_save_slots(nvwn_engine* e, const int* slots, int n, void* states, void* stream);
/* Slot slots[i] continues state i (states + i * nvwn_slot_state_bytes, host or device memory, 16-byte aligned) from the engine's
 * next sample t0: its history row is cleared and the state's inputs written at engine times t0 - d_l .. t0 - 1 (negative times
 * included), its fed-back indices set, its selector origin set to t0 - position and its key to the state's seed, so
 * nvwn_set_selectors_random_slots draws what the utterance would have drawn.  A per-slot call, as nvwn_restart_slots.  The first
 * such call at t0 < maxDil since nvwn_reset_history also zeroes the negative times of every slot and makes every launch read the
 * history at every step, as nvwn_prime_slots_from_score does.  Host states may be reused on return; device states are read in
 * order on `stream` (their headers are read before return).  Refused with NVWN_EINVAL, changing nothing: NULL arguments, a bad
 * slot list, a header whose tag, dtype, R, L or max_dilation differs from the engine's, or whose position or indices are out of
 * range.  That the state was made with the same weights is the caller's responsibility: nothing in it records them. */
int nvwn_load_slots(nvwn_engine* e, const int* slots, int n, const void* states, void* stream);
/* Prompted streams: the slot states of scored prompts.  With an open scoring stream of batch_size Bs and next sample P >= 1, writes
 * state i for scoring row rows[i] to states + i * nvwn_slot_state_bytes (host or device memory, 16-byte aligned), in the format of
 * nvwn_save_slots: dtype NVWN_FP16, position P, the row's codes of samples P - 2 and P - 1 as the fed-back indices, seed seeds[i]
 * (seeds NULL: 0), zero reserved fields, then each layer's inputs x_l of times [P - d_l, P) from the scorer's fronts, zeros before
 * time 0.  It is byte for byte the state nvwn_save_slots writes of a slot primed from that row by nvwn_prime_slots_from_score, so
 * nvwn_load_slots resumes the prompt in any slot of any fp16 engine of the same R, L and maxDil, and no engine has to keep rows or
 * store positions free for the scoring.  The scoring stream stays open and unchanged; nothing else changes.  Device states are
 * written asynchronously on `stream`; host states are complete on return.  Refused, changing nothing: no open scoring stream,
 * NULL arguments, n outside [1, Bs], rows outside [0, Bs) or given twice (NVWN_EINVAL); a packed stream (a row's fronts may hold
 * an earlier utterance's inputs) or an engine that is not NVWN_FP16 (NVWN_EUNSUPPORTED). */
int nvwn_score_save_states(nvwn_engine* e, const int* rows, int n, const unsigned long long* seeds, void* states, void* stream);

/* Multi-model serving: several models of one shape in one engine, each group of rows generating with its own weights, and each
 * scoring row scoring with its own.  Model 0 is the engine's own weights (the setters, nvwn_weight_blob and nvwn_weights_updated);
 * every generation kernel reads the weights of a row's group's model, and the scorer those of a scoring row's model
 * (nvwn_set_score_models); nothing else about a row changes.  Scope:
 *   - nvwn_prime_from_score and nvwn_prime_slots_from_score refuse (NVWN_EINVAL) a row or slot whose group runs another model than
 *     the one its scoring row was scored with;
 *   - slot states record no model, as they record no weights: loading one into a group that runs the right model is the caller's job. */
enum { NVWN_MAX_MODELS = 64 };
/* Copies src's weights (its blob, as uploaded) into model `model` (1 <= model < NVWN_MAX_MODELS) of e.  src is any engine on the
 * same device with the same dtype, R, S, A, L, max_dilation and tanh_embed (any B, N or kernel).  Later changes to src do not
 * reach e; calling again replaces the model.  Returns when src may be changed or destroyed.  Refused with NVWN_EINVAL, changing
 * nothing: NULL arguments, model 0 or an index out of range, a source of another shape, dtype, tanh_embed or device. */
int nvwn_set_model(nvwn_engine* e, int model, const nvwn_engine* src);
/* Rows per model group: rows [g*G, (g+1)*G) always run one model.  Fixed at creation by the kernel family: the latency kernels 8
 * when a full-batch run takes 8-utterance clusters, else 16; the tensor-core kernel its tile; the CUDA-core kernel 4. */
int nvwn_model_group(nvwn_engine* e, int* rows);
/* models[g] for each of the ceil(B / G) groups; every entry must be 0 or a model already set.  Stream-ordered on `stream`; takes
 * effect from the next launch.  Host array, copied before return.  Default: every group runs model 0, also after
 * nvwn_reset_history, which leaves the models and the table alone.  Refused with NVWN_EINVAL, changing nothing: NULL arguments,
 * n_groups != ceil(B / G), an entry naming a model that was never set. */
int nvwn_set_group_models(nvwn_engine* e, const int* models, int n_groups, void* stream);
/* Scoring by model: models[b] is the model scoring row b runs, for every b in [0, B) (n_rows = B); each entry 0 or a model already
 * set.  It applies to nvwn_score, nvwn_score_stream, nvwn_score_stream_packed and nvwn_score_save_states; a call of batch_size
 * Bs < B uses entries [0, Bs).  A row's logp, logits and state are, bit for bit, those an engine holding its model as model 0
 * gives the same utterance.  Rows are independent of the generation groups.  Host array, copied before return; the device copy
 * is made on `stream`, which the scoring calls must follow (one stream, or ordered).
 *   - Default: all 0, which runs the one-model scorer: every call gives the bits of an engine that never had a table.
 *   - Setting a table ends an open scoring stream (its fronts were computed with the old models), as nvwn_set_model of a model
 *     that one of the stream's rows runs does; nvwn_reset_history, generation calls and nvwn_set_group_models leave it alone.
 *   - Each model in use gets its own scorer image, packed on the first scoring call that runs it after a change, freed by
 *     nvwn_destroy (the size of model 0's: about 1.75 MB at R64 L20 S256, 7 MB at R128 L30).
 * Refused, changing nothing: NULL arguments, n_rows != B, an entry negative, >= NVWN_MAX_MODELS or never set (NVWN_EINVAL); an
 * engine that is not NVWN_FP16 (NVWN_EUNSUPPORTED). */
int nvwn_set_score_models(nvwn_engine* e, const int* models, int n_rows, void* stream);

/* last-sample activations [B][dim] as fp32 (nv_wavenet.cuh:424-438); valid after a run with dump=1 */
int nvwn_get_xt_out(nvwn_engine* e, int layer, float* out);
int nvwn_get_skip_out(nvwn_engine* e, int layer, float* out);
int nvwn_get_zs(nvwn_engine* e, float* out);
int nvwn_get_za(nvwn_engine* e, float* out);
int nvwn_get_p(nvwn_engine* e, float* out);

/* introspection: what the last launch used */
typedef struct {
    int kernel;            /* NVWN_KERNEL_STREAM / NVWN_KERNEL_TENSORCORE / NVWN_KERNEL_LATENCY */
    int grid, block, smem_bytes, batch_per_cta, cluster;
    unsigned long long launches;        /* kernel launches issued by this engine so far */
    unsigned long long weight_bytes;    /* algorithmic weight+bias bytes per utterance-sample (BASELINE.md §2) */
} nvwn_launch_info;
int nvwn_get_launch_info(nvwn_engine* e, nvwn_launch_info* info);
int nvwn_device_count(void);
int nvwn_set_device(int device);

#ifdef __cplusplus
}
#endif
#endif
