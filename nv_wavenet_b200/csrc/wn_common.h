// wn_common.h -- shared declarations of the WaveNet inference engine (host + device).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>

// Everything a kernel launch needs.  Device pointers only.
// Replaces nv_wavenet_params<T_weight,T_data> (nv_wavenet.cuh:40-85) of the reference.
struct WnParams {
    int L, R, S, A, maxDil;
    int B;              // batch size of this run (stride of Lh / selectors / ring, nv_wavenet.cuh:144)
    int N;              // num_samples of this run (row stride of yOut, singleblock.cuh:245)
    int init_sample, count;
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
};

struct WnLaunchInfo {
    int kernel, grid, block, smem_bytes, batch_per_cta, cluster;
};

// stream kernel (wn_stream_kernel.cu): CUDA-core, one CTA per batch tile, weights streamed from L2.
cudaError_t wn_launch_stream(const WnParams& p, int contract, cudaStream_t stream, WnLaunchInfo* info);   // 0 fp32 exact, 1 fp16, 2 fp32 fast
bool wn_stream_supported(int R, int S, int A, bool fp16);

// teacher-forced scoring (wn_score_kernel.cu, DESIGN.md §5.4): one time chunk of T steps x Bs utterances, rows m = (t - t0) * Bs + b
struct WnScoreChunk {
    int L, R, S, A, maxDil, tanhEmbed;
    int Bs, Be;                     // utterances scored / of the engine (stride of the conditioning chunk)
    int N, t0, T, Tcap;             // num_samples of the call (row stride of audio and logp), first step, steps, chunk capacity
    const void* image;              // scorer weight image (wn_score_pack)
    const void *embPrev, *embCur;   // fp16 [A][R] (engine blob)
    const int* audio;               // device [Bs][N]
    const float* lh;                // conditioning of the chunk, fp32 [T][L][Be][2R]
    __half* xh;                     // fp16 layer inputs; layer l at wn_score_xh_offset(l): [d_l * Bs history rows | T * Bs rows][R]
    float* xf;                      // fp32 residual stream [T * Bs][R]
    __half* H;                      // gate outputs [T * Bs][L * R]
    float* logp;                    // device [Bs][N]
    float* logits;                  // row (t, b) -> logits + b * logits_ld + (t - logits_t0) * A, or NULL
    long long logits_ld;
    int logits_t0;
};
int wn_score_dilation(int layer, int maxDil);
size_t wn_score_xh_offset(int layer, int L, int maxDil, int Tcap, int Be, int R);   // in elements; layer = L gives the total
size_t wn_score_image_bytes(int R, int S, int A, int L);
cudaError_t wn_score_pack(void* image, const WnParams& p, cudaStream_t stream);
cudaError_t wn_score_check_audio(const int* audio, size_t n, int A, unsigned long long* first_bad, cudaStream_t stream);
cudaError_t wn_score_chunk(const WnScoreChunk& c, cudaStream_t stream);

// conversions (wn_convert.cu)
cudaError_t wn_f32_to_f16(__half* dst, const float* src_dev, size_t n, cudaStream_t stream);
cudaError_t wn_f16_to_f32(float* dst, const __half* src_dev, size_t n, cudaStream_t stream);
cudaError_t wn_fill_selectors(float* dst, size_t n, unsigned long long seed, cudaStream_t stream);
cudaError_t wn_fill_int(int* dst, int value, size_t n, cudaStream_t stream);
