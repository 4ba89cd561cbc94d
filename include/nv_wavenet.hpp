/*
 * nv_wavenet.hpp -- C++ facade with the class surface of the reference's
 *   template <typename T_weight, typename T_data, int R=64, int S=128, int A=256> class nvWavenetInfer
 * (nv_wavenet.cuh:220-640) forwarding to the C-ABI of libwavenet_infer.so (include/nvwn_b200.h).
 *
 * The reference class is header-only and instantiates its kernels in the caller's translation unit;
 * this facade is plain host C++ (no nvcc needed): the sm_90a kernels are compiled once inside the
 * library for every supported (precision, R, S) and selected at run time.
 *
 *   T_weight / T_data : float / float  -> bit-exact fp32 path
 *                       half2 / half   -> fp16 tensor-core path
 *   Implementation    : the enum values of the reference are accepted; all map to the one kernel family.
 *   Errors            : CUDA / argument errors print "GPUassert: ..." and exit(code) like gpuErrChk
 *                       (nv_wavenet_util.cuh:34-40); launch failures make run*() return false.
 */
#ifndef NV_WAVENET_HPP
#define NV_WAVENET_HPP

#include <cuda_fp16.h>
#include <cuda_runtime_api.h>
#include <stdio.h>
#include <stdlib.h>

#include <vector>

#include "nvwn_b200.h"

namespace nvwn_detail {
template <typename T_data> struct dtype_of;
template <> struct dtype_of<float> { enum { value = NVWN_FP32 }; };
template <> struct dtype_of<half> { enum { value = NVWN_FP16 }; };
inline void check(int rc, const char* file, int line)
{
    if (rc != 0) {
        fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), file, line);
        exit(rc > 0 ? rc : 1);
    }
}
}  // namespace nvwn_detail
#define NVWN_CHK(x) nvwn_detail::check((x), __FILE__, __LINE__)

template <typename T_weight, typename T_data, int R = 64, int S = 128, int A = 256>
class nvWavenetInfer {
public:
    enum Implementation { AUTO = 0, SINGLE_BLOCK, DUAL_BLOCK, PERSISTENT, MANYBLOCK_NONPERSISTENT };

protected:
    nvwn_engine* m_engine;
    int m_maxBatch, m_maxSamples, m_num_samples_per_chunk;

public:
    nvWavenetInfer(int numLayers, int maxDilation, int batchSize, int numSamples, int impl = 0, bool tanhEmbed = true)
        : m_engine(NULL), m_maxBatch(batchSize), m_maxSamples(numSamples), m_num_samples_per_chunk(0)
    {
        NVWN_CHK(nvwn_create(&m_engine, nvwn_detail::dtype_of<T_data>::value, R, S, A, numLayers, maxDilation,
                             batchSize, numSamples, impl, tanhEmbed ? 1 : 0));
    }
    virtual ~nvWavenetInfer() { nvwn_destroy(m_engine); }

    virtual void setEmbeddings(float* embedPrev, float* embedCur) { NVWN_CHK(nvwn_set_embeddings(m_engine, embedPrev, embedCur)); }
    virtual void setLayerWeights(int layer, float* Wprev, float* Wcur, float* Bh, float* Wres, float* Bres, float* Wskip, float* Bskip)
    {
        NVWN_CHK(nvwn_set_layer_weights(m_engine, layer, Wprev, Wcur, Bh, Wres, Bres, Wskip, Bskip));
    }
    virtual void setOutWeights(float* Wzs, float* Bzs, float* Wza, float* Bza) { NVWN_CHK(nvwn_set_out_weights(m_engine, Wzs, Bzs, Wza, Bza)); }
    void setInputs(float* Lh, float* outputSelectors) { NVWN_CHK(nvwn_set_inputs(m_engine, Lh, outputSelectors)); }

    void getXtOut(int layer, float* hXt) { NVWN_CHK(nvwn_get_xt_out(m_engine, layer, hXt)); }
    void getSkipOut(int layer, float* hSkipOut) { NVWN_CHK(nvwn_get_skip_out(m_engine, layer, hSkipOut)); }
    void getZs(float* hZs) { NVWN_CHK(nvwn_get_zs(m_engine, hZs)); }
    void getZa(float* hZa) { NVWN_CHK(nvwn_get_za(m_engine, hZa)); }
    void getP(float* hP) { NVWN_CHK(nvwn_get_p(m_engine, hP)); }
    void getYOut(int* yOut, int offset, int size, cudaStream_t stream = 0) { NVWN_CHK(nvwn_get_yout(m_engine, yOut, offset, size, stream)); }
    /* Not in the reference class: mu-law decoded audio of yOut[b][offset .. offset+size) for every b, on the device
     * (replaces the host post-processing of pytorch/nv_wavenet_inference.py:55-60); see nvwn_get_audio. */
    void getAudio(float* audio_f32, short* audio_i16, int offset, int size, bool saturate = false, cudaStream_t stream = 0)
    {
        NVWN_CHK(nvwn_get_audio(m_engine, audio_f32, audio_i16, offset, size, saturate ? 1 : 0, stream));
    }

    /* Chunked generation with overlapped device->host copies of finished chunks (nv_wavenet.cuh:445-497).
     * consume(yOut, initSample, count) is called per chunk once its copy has landed. */
    template <class Callback>
    bool run_chunks(int num_samples_per_chunk, Callback consume, int num_samples, int batch_size, int* yOut = NULL,
                    int batch_size_per_block = 1, bool dumpActivations = false, cudaStream_t stream = 0)
    {
        bool result = true;
        cudaStream_t stream_compute = stream, stream_copy;
        if (!stream) cudaStreamCreate(&stream_compute);
        cudaStreamCreate(&stream_copy);
        const int num_chunks = (num_samples + num_samples_per_chunk - 1) / num_samples_per_chunk;
        std::vector<cudaEvent_t> ev_compute(num_chunks), ev_copy(num_chunks);
        for (int j = 0; j < num_chunks; j++) {
            cudaEventCreateWithFlags(&ev_compute[j], cudaEventDisableTiming);
            cudaEventCreateWithFlags(&ev_copy[j], cudaEventDisableTiming);
        }
        for (int j = 0; j < num_chunks; j++) {
            const int init = j * num_samples_per_chunk;
            m_num_samples_per_chunk = (j == num_chunks - 1) ? num_samples - init : num_samples_per_chunk;
            result = result && run_partial(init, num_samples, batch_size, NULL, batch_size_per_block, true, stream_compute);
            cudaEventRecord(ev_compute[j], stream_compute);
            cudaStreamWaitEvent(stream_copy, ev_compute[j], 0);
            if (yOut != NULL) getYOut(yOut, init, m_num_samples_per_chunk, stream_copy);
            cudaEventRecord(ev_copy[j], stream_copy);
        }
        for (int j = 0; j < num_chunks; j++) {
            const int init = j * num_samples_per_chunk;
            const int n = (j == num_chunks - 1) ? num_samples - init : num_samples_per_chunk;
            cudaEventSynchronize(ev_copy[j]);
            consume(yOut, init, n);
        }
        m_num_samples_per_chunk = 0;
        for (int j = 0; j < num_chunks; j++) { cudaEventDestroy(ev_compute[j]); cudaEventDestroy(ev_copy[j]); }
        if (stream != stream_compute) cudaStreamDestroy(stream_compute);
        cudaStreamDestroy(stream_copy);
        return result;
    }

    bool run_partial(int init_sample, int num_samples, int batch_size, int* yOut = NULL, int batch_size_per_block = 1,
                     bool dumpActivations = false, cudaStream_t stream = 0)
    {
        (void)batch_size_per_block;      /* the batch tile per CTA is chosen by the library */
        const int count = m_num_samples_per_chunk ? m_num_samples_per_chunk : num_samples;
        const int rc = nvwn_run_partial(m_engine, init_sample, count, num_samples, batch_size, yOut, dumpActivations ? 1 : 0, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }

    /* Not in the reference class: streaming generation of absolute samples [first_sample, first_sample + count) through the
     * engine's numSamples buffers used as rings, continuing from the last generation; see nvwn_run_stream. */
    bool run_stream(long long first_sample, int count, int batch_size, bool dumpActivations = false, cudaStream_t stream = 0)
    {
        const int rc = nvwn_run_stream(m_engine, first_sample, count, batch_size, dumpActivations ? 1 : 0, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }

    /* Not in the reference class: continuous batching over the rows of a streaming engine (slots); see nvwn_restart_slots,
     * nvwn_set_conditioning_slots and nvwn_set_selectors_random_slots. */
    bool restart_slots(const int* slots, int n, const unsigned long long* seeds = NULL, cudaStream_t stream = 0)
    {
        const int rc = nvwn_restart_slots(m_engine, slots, n, seeds, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }
    bool set_conditioning_slots(const float* Lh, const int* slots, int n, long long first_sample, int num_samples, cudaStream_t stream = 0)
    {
        const int rc = nvwn_set_conditioning_slots(m_engine, Lh, slots, n, first_sample, num_samples, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }
    bool set_selectors_random_slots(long long first_sample, int num_samples, cudaStream_t stream = 0)
    {
        const int rc = nvwn_set_selectors_random_slots(m_engine, first_sample, num_samples, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }

    /* Not in the reference class: each slot's conditioning produced on the device from its own utterance's mel frames; see
     * nvwn_cond_producer_set_weights, nvwn_cond_producer_set_slots and nvwn_cond_producer_run_slots. */
    bool cond_producer_set_weights(int n_cond_channels, const float* upsample_weight, const float* upsample_bias, int window, int stride,
                                   const float* cond_weight, const float* cond_bias, cudaStream_t stream = 0)
    {
        const int rc = nvwn_cond_producer_set_weights(m_engine, n_cond_channels, upsample_weight, upsample_bias, window, stride, cond_weight,
                                                      cond_bias, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }
    bool cond_producer_set_slots(const int* slots, int n, const float* const* features, const int* num_frames, const long long* starts,
                                 cudaStream_t stream = 0)
    {
        const int rc = nvwn_cond_producer_set_slots(m_engine, slots, n, features, num_frames, starts, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }
    bool cond_producer_run_slots(const int* slots, int n, long long first_sample, int num_samples, cudaStream_t stream = 0)
    {
        const int rc = nvwn_cond_producer_run_slots(m_engine, slots, n, first_sample, num_samples, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }

    /* Not in the reference class: live frames for single slots, each slot's utterance fed from a ring of its own; see
     * nvwn_cond_producer_open_live_slots, nvwn_cond_producer_attach_live and nvwn_cond_producer_push_slots. */
    bool cond_producer_open_live_slots(int ring_frames, cudaStream_t stream = 0)
    {
        const int rc = nvwn_cond_producer_open_live_slots(m_engine, ring_frames, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }
    bool cond_producer_attach_live(const int* slots, int n, const long long* starts, const int* first_frames, const float* const* features,
                                   const int* num_frames, cudaStream_t stream = 0)
    {
        const int rc = nvwn_cond_producer_attach_live(m_engine, slots, n, starts, first_frames, features, num_frames, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }
    bool cond_producer_push_slots(const int* slots, int n, const float* const* features, const int* num_frames, cudaStream_t stream = 0)
    {
        const int rc = nvwn_cond_producer_push_slots(m_engine, slots, n, features, num_frames, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }

    /* Not in the reference class: live vocoding, mel frames pushed as they arrive into a ring of ring_frames frames per utterance and
     * each sample's conditioning produced once its frames are in; see nvwn_cond_producer_open_live, nvwn_cond_producer_push and
     * nvwn_cond_producer_run_stream. */
    bool cond_producer_open_live(int n_cond_channels, const float* upsample_weight, const float* upsample_bias, int window, int stride,
                                 const float* cond_weight, const float* cond_bias, int ring_frames, cudaStream_t stream = 0)
    {
        const int rc = nvwn_cond_producer_open_live(m_engine, n_cond_channels, upsample_weight, upsample_bias, window, stride, cond_weight,
                                                    cond_bias, ring_frames, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }
    bool cond_producer_push(const float* features, int num_frames, cudaStream_t stream = 0)
    {
        const int rc = nvwn_cond_producer_push(m_engine, features, num_frames, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }
    bool cond_producer_run_stream(long long sample_begin, int sample_count, cudaStream_t stream = 0)
    {
        const int rc = nvwn_cond_producer_run_stream(m_engine, sample_begin, sample_count, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }

    /* Not in the reference class: teacher-forced scoring, logp[b * num_samples + t] = log p(audio[b][t] | audio[b][0..t),
     * conditioning) for every step at once, and optionally the fp32 logits; see nvwn_score.  fp16 engines only. */
    bool score(const int* audio, int num_samples, int batch_size, float* logp, float* logits = NULL, cudaStream_t stream = 0)
    {
        const int rc = nvwn_score(m_engine, audio, num_samples, batch_size, logp, logits, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }
    /* Not in the reference class: score of absolute samples [first_sample, first_sample + count) of audio of any length, continuing
     * the scoring stream (first_sample = 0 starts one); audio, logp and logits cover this call's samples only.  See nvwn_score_stream. */
    bool score_stream(const int* audio, long long first_sample, int count, int batch_size, float* logp, float* logits = NULL, cudaStream_t stream = 0)
    {
        const int rc = nvwn_score_stream(m_engine, audio, first_sample, count, batch_size, logp, logits, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }
    /* Not in the reference class: score_stream of a queue of utterances packed end to end in the rows; starts[b * count + i] != 0
     * begins a new utterance in row b at sample first_sample + i.  See nvwn_score_stream_packed. */
    bool score_stream_packed(const int* audio, const unsigned char* starts, long long first_sample, int count, int batch_size, float* logp,
                             float* logits = NULL, cudaStream_t stream = 0)
    {
        const int rc = nvwn_score_stream_packed(m_engine, audio, starts, first_sample, count, batch_size, logp, logits, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }
    /* Not in the reference class: after score_stream over a prompt [0, P), generation continues it from sample P (run_stream of
     * the scoring stream's batch_size).  See nvwn_prime_from_score. */
    bool prime_from_score(cudaStream_t stream = 0)
    {
        const int rc = nvwn_prime_from_score(m_engine, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }
    /* Not in the reference class: after score_stream over prompts [0, P), slot slots[i] continues scoring row rows[i] from the engine's
     * next sample.  See nvwn_prime_slots_from_score. */
    bool prime_slots_from_score(const int* rows, const int* slots, int n, const unsigned long long* seeds = NULL, cudaStream_t stream = 0)
    {
        const int rc = nvwn_prime_slots_from_score(m_engine, rows, slots, n, seeds, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }

    /* Not in the reference class: park slots and resume them in any slot of any engine of the same dtype, R, L and maxDil.
     * slot_state_bytes is the size of one state (0 on failure); see nvwn_save_slots and nvwn_load_slots. */
    unsigned long long slot_state_bytes()
    {
        unsigned long long bytes = 0;
        if (nvwn_slot_state_bytes(m_engine, &bytes) != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return bytes;
    }
    bool save_slots(const int* slots, int n, void* states, cudaStream_t stream = 0)
    {
        const int rc = nvwn_save_slots(m_engine, slots, n, states, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }
    bool load_slots(const int* slots, int n, const void* states, cudaStream_t stream = 0)
    {
        const int rc = nvwn_load_slots(m_engine, slots, n, states, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }
    /* Not in the reference class: the slot states of scoring rows rows[0..n) of the open scoring stream at its next sample P, for
     * load_slots on any compatible engine.  See nvwn_score_save_states. */
    bool score_save_states(const int* rows, int n, const unsigned long long* seeds, void* states, cudaStream_t stream = 0)
    {
        const int rc = nvwn_score_save_states(m_engine, rows, n, seeds, states, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }
    /* Not in the reference class: multi-model serving.  set_model copies src's weights into model `model` (1 <= model <
     * NVWN_MAX_MODELS) of this engine; model_group is the rows G per model group (0 on failure); set_group_models gives each of the
     * ceil(B / G) groups its model from the next launch on `stream`.  See nvwn_set_model, nvwn_model_group and nvwn_set_group_models. */
    bool set_model(int model, const nvWavenetInfer& src)
    {
        const int rc = nvwn_set_model(m_engine, model, src.m_engine);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }
    int model_group()
    {
        int rows = 0;
        if (nvwn_model_group(m_engine, &rows) != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rows;
    }
    bool set_group_models(const int* models, int n_groups, cudaStream_t stream = 0)
    {
        const int rc = nvwn_set_group_models(m_engine, models, n_groups, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }
    /* Scoring by model: models[b] is the model scoring row b runs, for each of the B rows (n_rows = B).  See nvwn_set_score_models. */
    bool set_score_models(const int* models, int n_rows, cudaStream_t stream = 0)
    {
        const int rc = nvwn_set_score_models(m_engine, models, n_rows, stream);
        if (rc != 0) fprintf(stderr, "GPUassert: %s %s %d\n", nvwn_last_error(), __FILE__, __LINE__);
        return rc == 0;
    }

    bool run(int num_samples, int batch_size, int* yOut = NULL, int batch_size_per_block = 1, bool dumpActivations = false,
             cudaStream_t stream = 0)
    {
        m_num_samples_per_chunk = 0;
        return run_partial(0, num_samples, batch_size, yOut, batch_size_per_block, dumpActivations, stream);
    }
};

#endif
