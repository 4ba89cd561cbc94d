// wn_common.h -- shared declarations of the WaveNet inference engine (host + device).
#pragma once
#include "../../include/nvwn_b200.h"
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>

// An engine's sizes and its kernel choice, both fixed by nvwn_create (wn_engine.cu, resolve_config) from its arguments and the
// environment switches of INTEGRATION.md §1.  Together they fix the layouts of the conditioning store, the history ring and the
// weight image.
struct WnConfig {
    int dtype, R, S, A, L, maxDil, B, N;    // B, N: what the engine holds; a run may take fewer
    int kernel;                             // NVWN_KERNEL_STREAM | NVWN_KERNEL_TENSORCORE | NVWN_KERNEL_LATENCY
    int tc_tile;                            // tensor-core: utterances per tile, 32 | 64 | 128
    bool tc_fused;                          // tensor-core: the fused schedule
    bool lat_cluster;                       // latency: the three-CTA cluster kernel may run
    int stream_bt;                          // stream: utterances per CTA, 1 | 2 | 4; 0 = chosen from the run's batch
    bool stream_ring;                       // stream, fp32: the weights may go through the shared-memory ring
};

// One model's weights on the device: its blob, laid out as the engine's, and its family's image (NULL: the family reads the blob)
struct WnModel {
    const char* blob;
    const void* image;
};

// Everything a kernel launch needs.  Device pointers only.
// Replaces nv_wavenet_params<T_weight,T_data> (nv_wavenet.cuh:40-85) of the reference.
struct WnParams {
    int L, R, S, A, maxDil;
    int B;              // batch size of this run (stride of Lh / selectors / ring, nv_wavenet.cuh:144)
    int N;              // num_samples of this run (row stride of yOut, singleblock.cuh:245)
    int init_sample, count;                             // buffer positions: Lh, sel, forced and yOut rows (see ring_slot)
    int tanhEmbed, dump;
    // model (TD = float in fp32 mode, __half in fp16 mode)
    const void *embPrev, *embCur;                       // TD [A][R]
    const void *Wprev, *Wcur, *Wres, *Wskip;            // TD col-major, [L][M*K]
    const void *Wzs, *Wza;                              // TD col-major A x S, A x A
    const void *Bh, *Bres, *Bskip, *Bzs, *Bza;          // TD [L][2R], [L][R], [L][S], [A], [A]
    // inputs
    const void* Lh;                                     // TD [N][L][B][2R]
    const float* sel;                                   // [N][B]
    const int* forced;                                  // [B][N] or NULL
    // state
    int *yPrev, *yCur;                                  // [B]
    void* ring;                                         // TD [(maxDil+1)][L][B][R]  layer inputs
    int* yOut;                                          // [B][N]
    // last-sample activation dumps (fp32)
    float *xtOut, *skipOut, *Zs, *Za, *P;               // [L][B][R], [L][B][S], [B][A] x3
    // optional timeline trace of one sample (debug): 3 x 1024 (tag << 48 | clock) words, or NULL
    unsigned long long* trace;
    int trace_t;
    // Absolute time of step init_sample, for the history only (the buffers are rings in streaming use, DESIGN.md §6):
    int ring_slot;      // its history-ring slot, t mod (maxDil+1)
    int hist_t;         // t clamped to maxDil: x_l[t-d] exists iff hist_t + (step - init_sample) >= d, and d <= maxDil
    // Model groups (nvwn_set_group_models, DESIGN.md §6): rows [g * group_rows, (g + 1) * group_rows) run model group_model[g]
    // (device [ceil(B / group_rows)]), whose blob and image are models[group_model[g]] (device [NVWN_MAX_MODELS]).  The model
    // pointers above and the launch's image are model 0's.  group_model NULL: every row runs them, and no kernel looks anything up.
    int group_rows;
    const int* group_model;
    const WnModel* models;
};

#ifdef __CUDACC__
// The weights a CTA or cluster whose first row is `row` runs with p.group_model set: every blob pointer of p moved by `shift`
// bytes, from model 0's blob to its group's model's, and that model's image.  Read once, at kernel entry.
struct WnGroupWeights {
    long long shift;
    const unsigned char* image;
    template <typename T> __device__ __forceinline__ const T* at(const void* q) const
    {
        return reinterpret_cast<const T*>(static_cast<const char*>(q) + shift);
    }
};
__device__ __forceinline__ WnGroupWeights wn_group_weights(const WnParams& p, int row)
{
    const WnModel m = p.models[p.group_model[row / p.group_rows]];
    return {(long long)(m.blob - p.models[0].blob), static_cast<const unsigned char*>(m.image)};
}
#endif

// p with its first k steps dropped (a launch split into pieces)
inline WnParams wn_params_skip(WnParams p, int k)
{
    p.init_sample += k;
    p.count -= k;
    p.ring_slot = (p.ring_slot + k) % (p.maxDil + 1);
    p.hist_t = p.hist_t + k < p.maxDil ? p.hist_t + k : p.maxDil;
    return p;
}

struct WnLaunchInfo {
    int kernel, grid, block, smem_bytes, batch_per_cta, cluster;
};

// One kernel family as the engine sees it: the sizes of its conditioning store, history ring and weight image, the conversions of
// the store, and the launch.  The engine picks one at creation.  Conditioning enters and leaves the store as fp32 [n][L][B][2R]
// in device memory; the plain fp32 store also copies from host memory.
struct WnFamily {
    size_t (*store_bytes)(const WnConfig& c);       // c.N samples of conditioning
    size_t (*ring_bytes)(const WnConfig& c);
    size_t (*image_bytes)(const WnConfig& c);       // NULL when pack is
    cudaError_t (*convert)(const WnConfig& c, void* store, const float* src, int first_sample, int num_samples, cudaStream_t stream);
    cudaError_t (*readback)(const WnConfig& c, float* dst_dev, const void* store, int first_sample, int num_samples, cudaStream_t stream);
    // Per-utterance-row operations (continuous batching, DESIGN.md §6), rows_dev: n distinct rows in [0, c.B), device memory.
    // wn_layout.cuh implements these and the history writers once, over each family's layout.
    // clear_rows zeroes every byte of rows rows_dev[i] in all (maxDil+1) x L history-ring entries and no other byte;
    // convert_rows converts fp32 [num_pos][L][n][2R] (device) into rows rows_dev[i] of store positions [first_pos, +num_pos),
    // bit for bit as convert does, and leaves every other row alone.
    cudaError_t (*clear_rows)(const WnConfig& c, void* ring, const int* rows_dev, int n, cudaStream_t stream);
    cudaError_t (*convert_rows)(const WnConfig& c, void* store, const float* src, const int* rows_dev, int n, int first_pos, int num_pos,
                                cudaStream_t stream);
    // History writers (priming from a scoring stream, DESIGN.md §5.4).  put_history writes fp16 src [n][batch][R] (device), the
    // values x_layer[t] of absolute times [t_first, t_first + n), n <= maxDil + 1, rows 0..batch-1, into ring slot t mod (maxDil+1)
    // of that layer, where a run of batch_size = batch reads them, and no other byte; get_history (debug) reads the whole ring back
    // as fp32 [(maxDil+1)][L][batch][R] (device), slot by slot, at that stride, or with rows_dev (device, batch rows in [0, c.B))
    // those rows at the engine's batch stride.
    cudaError_t (*put_history)(const WnConfig& c, void* ring, const __half* src, int layer, long long t_first, int n, int batch, cudaStream_t stream);
    cudaError_t (*get_history)(const WnConfig& c, float* dst, const void* ring, int batch, const int* rows_dev, cudaStream_t stream);
    // Per-slot history writers and reader (priming single slots, parking and resuming them, DESIGN.md §6), at the engine's batch
    // stride, for absolute times t that may be negative, in ring slot ((t mod M) + M) mod M, M = maxDil + 1.  A row's values are
    // in the ring's element type (fp16 on NVWN_FP16 engines, else fp32) in device memory: the value of time t_first + j of source
    // row i at element src_row(i) * row_pitch + j * time_pitch, src_row(i) = src_rows_dev[i] (src_rows_dev NULL: i); both pitches
    // are multiples of 8 elements, and the base 16-byte aligned.  put_history_rows writes the values x_layer[t] of times [t_first,
    // t_first + n_t), n_t <= M, into ring rows rows_dev[i] (n distinct rows in [0, c.B)), and no other byte; get_history_rows
    // reads them back into dst at the same addresses, src_row(i) = i, writing zeros for the times before origin_dev[rows_dev[i]];
    // clear_times zeroes rows 0..c.B-1 of every layer's entries of times [t_first, t_first + n_t), n_t <= M, and no other byte.
    cudaError_t (*put_history_rows)(const WnConfig& c, void* ring, const void* src, const int* src_rows_dev, size_t row_pitch, size_t time_pitch,
                                    const int* rows_dev, int n, int layer, long long t_first, int n_t, cudaStream_t stream);
    cudaError_t (*get_history_rows)(const WnConfig& c, const void* ring, void* dst, size_t row_pitch, size_t time_pitch, const int* rows_dev, int n,
                                    int layer, long long t_first, int n_t, const long long* origin_dev, cudaStream_t stream);
    cudaError_t (*clear_times)(const WnConfig& c, void* ring, long long t_first, int n_t, cudaStream_t stream);
    cudaError_t (*pack)(void* image, const WnParams& p, cudaStream_t stream);      // weight blob -> image; NULL: the kernels read the blob
    cudaError_t (*launch)(const WnConfig& c, const WnParams& p, const void* image, cudaStream_t stream, WnLaunchInfo* info);
    bool whole_batch;                               // a run must take all c.B utterances
    // rows per model group (WnParams::group_rows): a multiple of the rows every CTA or cluster of any run of the engine serves
    int (*group_rows)(const WnConfig& c);
};
extern const WnFamily wn_stream_family;             // wn_stream_kernel.cu: CUDA-core, one CTA per batch tile, weights streamed from L2
extern const WnFamily wn_tc_family;                 // wn_tc_kernel.cu: fp16 tensor-core (wgmma) kernel
extern const WnFamily wn_lat_family;                // wn_lat_kernel.cu: fp16 latency-mode kernels
bool wn_stream_supported(int R, int S, int A, bool fp16);
bool wn_tc_supported(int R, int S, int A, int L, int B);
bool wn_lat_supported(int R, int S, int A, int L);
int wn_lat_max_clusters(int S, int rows);          // three-CTA clusters of `rows` (8 or 16) utterances the device runs at once

// the plain conditioning store of the stream kernel, [N][L][B][2R], fp16 on NVWN_FP16 engines, else fp32: whole-store conversions
// (wn_convert.cu)
cudaError_t wn_plain_convert(const WnConfig& c, void* store, const float* src, int first_sample, int num_samples, cudaStream_t stream);
cudaError_t wn_plain_readback(const WnConfig& c, float* dst_dev, const void* store, int first_sample, int num_samples, cudaStream_t stream);

// Scoring by model (nvwn_set_score_models, DESIGN.md §5.5): the rows b < Bs of a call grouped by model.  Segment k holds the n[k]
// rows order[first[k] .. first[k] + n[k]) (ascending) of model model[k], segments by model.  In a chunk of T steps its T * n[k] local
// rows q go to the chunk's row m = (q / n[k]) * Bs + order[first[k] + q % n[k]], and they make ceil(T * n[k] / 64) tiles of one
// model, the segments' tiles in order.  image[v], embPrev[v] and embCur[v] are model v's score image and embeddings.
struct WnScoreSegs {
    int count;
    int model[NVWN_MAX_MODELS], n[NVWN_MAX_MODELS], first[NVWN_MAX_MODELS];
    const void* image[NVWN_MAX_MODELS];
    const void *embPrev[NVWN_MAX_MODELS], *embCur[NVWN_MAX_MODELS];
    const int* order;               // device: every row of the table by model, then by row; a call's rows of a model are a prefix
    const int* row_model;           // device [Be]: the model of row b
};

// teacher-forced scoring (wn_score_kernel.cu, DESIGN.md §5.4): one time chunk of T steps x Bs utterances, rows m = (t - t0) * Bs + b
struct WnScoreChunk {
    int L, R, S, A, maxDil, tanhEmbed;
    int Bs, Be;                     // utterances scored / of the engine (stride of the conditioning chunk)
    int N, t0, T, Tcap;             // num_samples of the call (row stride of audio and logp), first step, steps, chunk capacity
    const void* image;              // scorer weight image (wn_score_pack)
    const void *embPrev, *embCur;   // fp16 [A][R] (engine blob)
    const int* audio;               // device [Bs][N]
    const int* codes;               // device [Bs][2]: the codes of steps -2 and -1 of the call (128, 128 at a fresh start)
    const float* lh;                // conditioning of the chunk, fp32 [T][L][Be][2R]
    __half* xh;                     // fp16 layer inputs; layer l at wn_score_xh_offset(l): [d_l * Bs history rows | T * Bs rows][R]
    float* xf;                      // fp32 residual stream [T * Bs][R]
    __half* H;                      // gate outputs [T * Bs][L * R]
    float* logp;                    // device [Bs][N]
    float* logits;                  // row (t, b) -> logits + b * logits_ld + (t - logits_t0) * A, or NULL
    long long logits_ld;
    int logits_t0;
    // packed scoring (nvwn_score_stream_packed), or starts NULL: the call's start flags, device [Bs][N]; the chunk's local times
    // [T][Bs] are made in tau from the per-row carry tau_carry [Bs], which moves on to the sample after the chunk
    const unsigned char* starts;
    int* tau;
    int* tau_carry;
    // scoring by model, or NULL: every row runs `image` and the blob's embeddings.  segs is the host copy, segs_dev the same bytes
    // on the device, which the kernels read
    const WnScoreSegs* segs;
    const WnScoreSegs* segs_dev;
};
int wn_score_dilation(int layer, int maxDil);
size_t wn_score_xh_offset(int layer, int L, int maxDil, int Tcap, int Be, int R);   // in elements; layer = L gives the total
size_t wn_score_image_bytes(int R, int S, int A, int L);
cudaError_t wn_score_pack(void* image, const WnParams& p, cudaStream_t stream);
cudaError_t wn_score_check_audio(const int* audio, size_t n, int A, unsigned long long* first_bad, cudaStream_t stream);
cudaError_t wn_score_chunk(const WnScoreChunk& c, cudaStream_t stream);
// streaming scoring: codes [Bs][2] <- the codes of steps count-2 and count-1 of a call's audio [Bs][N] (count = 1: the pair shifts by one)
cudaError_t wn_score_carry_codes(int* codes, const int* audio, int N, int count, int Bs, cudaStream_t stream);

// conversions (wn_convert.cu)
cudaError_t wn_f32_to_f16(__half* dst, const float* src_dev, size_t n, cudaStream_t stream);
cudaError_t wn_f16_to_f32(float* dst, const __half* src_dev, size_t n, cudaStream_t stream);
cudaError_t wn_fill_selectors(float* dst, size_t n, unsigned long long seed, unsigned long long first, cudaStream_t stream);
cudaError_t wn_fill_int(int* dst, int value, size_t n, cudaStream_t stream);
// per-slot selectors: dst[p * B + b], p in [0, n), = the selector of counter first_t + p - origin[b] under key seed[b]
cudaError_t wn_fill_selectors_slots(float* dst, int n, int B, long long first_t, const long long* origin, const unsigned long long* seed,
                                    cudaStream_t stream);
// restart of rows rows[0..n): yPrev = yCur = 128, origin = t0, seed = seeds[i] (seeds NULL: 0)
cudaError_t wn_restart_rows(const int* rows, int n, const unsigned long long* seeds, long long t0, int* yPrev, int* yCur, long long* origin,
                            unsigned long long* seed, cudaStream_t stream);
// fed-back indices of rows b < n from a scoring stream's codes [n][2] (the codes of steps t-2 and t-1 of its next sample t):
// yPrev[b] = codes[b][0], yCur[b] = codes[b][1]
cudaError_t wn_feedback_from_codes(const int* codes, int n, int* yPrev, int* yCur, cudaStream_t stream);
// state of slots slots[0..n) primed from scoring rows rows[i]: yPrev = codes[rows[i]][0], yCur = codes[rows[i]][1], origin = t_origin,
// seed = seeds[i] (seeds NULL: 0)
cudaError_t wn_prime_rows(const int* codes, const int* rows, const int* slots, int n, const unsigned long long* seeds, long long t_origin, int* yPrev,
                          int* yCur, long long* origin, unsigned long long* seed, cudaStream_t stream);
// A saved slot state (nvwn_save_slots) starts with this header; wn_slot_state_bytes gives the whole blob
static_assert(sizeof(nvwn_slot_state_header) == 64, "the slot state header is 64 bytes");
size_t wn_slot_state_bytes(const WnConfig& c);
// headers of the states at states + i * bytes for slots rows[i]: the engine's sizes, position next_t - origin[rows[i]], seed and
// fed-back indices of the slot
cudaError_t wn_save_slot_scalars(void* states, size_t bytes, const int* rows, int n, const WnConfig& c, long long next_t, const int* yPrev,
                                 const int* yCur, const long long* origin, const unsigned long long* seed, cudaStream_t stream);
// the states of scoring rows rows[0..n) of an open stream of next sample P, at states + i * bytes (nvwn_score_save_states): the
// fp16 header of the engine's sizes with position P, codes[rows[i]] as the fed-back indices and seeds[i] (NULL: 0), then each
// layer's front rows of rows[i], read from the scoring scratch's xh (chunk capacity Tcap, engine batch Be, stream batch Bs)
cudaError_t wn_score_save_states(void* states, size_t bytes, const __half* xh, const int* codes, const int* rows, int n, const unsigned long long* seeds,
                                 const WnConfig& c, long long P, int Tcap, int Be, int Bs, cudaStream_t stream);
// the reverse for a load at engine time t0: slot rows[i] takes state i's fed-back indices and seed, and origin t0 - position
cudaError_t wn_load_slot_scalars(const void* states, size_t bytes, const int* rows, int n, long long t0, int* yPrev, int* yCur, long long* origin,
                                 unsigned long long* seed, cudaStream_t stream);
cudaError_t wn_mulaw_decode(const int* yOut, int N, int offset, int size, int B, int A, const float* lut_f, const short* lut_s, float* out_f,
                            short* out_s, cudaStream_t stream);

// conditioning producer (wn_cond_producer.cu)
cudaError_t wn_cond_transpose_wu(float* WuT, const float* Wu, int C, int K, cudaStream_t stream);
void wn_cond_host(float* Lh, const float* feat, const float* Wu, const float* bu, const float* Wc, const float* bc,
                  int B, int C, int T, int K, int stride, int L, int R);
// row i of a chunk is the utterance with frames [C][T] at frames + foff whose sample 0 is absolute sample start; in a live sequence
// (DESIGN.md §6) its frames are a ring [C][ring] there instead, frame m at column m mod ring, and T counts the frames pushed so far
struct WnCondSlot {
    long long foff, start;
    int T, ring;
};
// out [m][L][k][2R] for absolute samples [n0, n0 + m) of the k utterances in tab (device); with `mask`, zero at or past each one's
// end (without it the caller knows no utterance ends before n0 + m); with `ring`, the rows' frames are rings and the caller has
// checked that every frame the samples read is still in them; U scratch holds k * m * C floats
cudaError_t wn_cond_produce_slots(float* out, float* U, const float* frames, const WnCondSlot* tab, const float* WuT, const float* bu, const float* Wc,
                                  const float* bc, int k, int C, int K, int stride, int L, int R, long long n0, int m, bool mask, bool ring,
                                  cudaStream_t stream);
