// wn_cond_producer.cu -- conditioning producer (SURVEY.md 8f next-2): local-conditioning features (mel frames) ->
// Lh[n][l][b][2R] on the device, in chunks of whole samples that go straight into the engine's conditioning store
// (the kernel family's convert / convert_rows), so the [N][L][B][2R] fp32 tensor of the reference (10.5 GB for C3) never exists.
//
// Replaces, for inference, WaveNet.get_cond_input (pytorch/wavenet.py:190-202) and the permutes that follow it
// (pytorch/nv_wavenet.py:48-49,181):
//     u = ConvTranspose1d(C, C, window, stride)(features)[:, :, :-(window - stride)]      -> [B][C][T * stride]
//     y = Conv1d(C, L * 2R, 1)(u)                                                       -> [B][L * 2R][T * stride]
//     Lh[n][l][b][c] = y[b][l * 2R + c][n]
// Two stages (the composed operator would need C * window * L * 2R weights).  The arithmetic of one output element
// lives in __host__ __device__ functions that the host reference below (nvwn_cond_from_features_host, used by the CPU
// tests against vectors generated from the reference's own module) and the kernels share.
// fp32 FMA, every output element accumulated in the order of the shared element functions (so host reference, simple kernels
// and the tiled kernel below agree bit for bit).  The projection is 94 % of the flops (C3: 0.42 TFLOP per 16000 samples x 64
// utterances): a register-tiled kernel (128 x 128 outputs per CTA, 8 x 8 per thread, operands through shared memory).
// One producer serves the whole-batch and the per-slot calls: each of the k rows of a chunk reads its own utterance's frames at its
// own sample offset through a small table (for a whole batch, row b's frames are features[b] and its start is 0); the projection
// is one kernel with B = k.
#include "wn_common.h"

namespace {

// u[b][co][n] of the trimmed transposed convolution.  features [B][C][T], Wu [C_in][C_out][K] (torch ConvTranspose1d
// layout) or, with WU_T, its [K][C_in][C_out] transpose (coalesced across co).  out[n] += in[m] * W[k] for m*stride + k = n.
// With RING the frames are a ring [B][C][F] (F = ring): frame m at column m mod F.  Either way sample n reads frames
// ceil((n - K + 1) / stride) .. floor(n / stride), in that order from the last, so its value is fixed once frame floor(n / stride) is in.
template <bool WU_T, bool RING = false>
__host__ __device__ inline float upsample_element(const float* __restrict__ feat, const float* __restrict__ Wu, const float* __restrict__ bu,
                                                  int C, int T, int K, int stride, int b, int co, int n, int ring = 0)
{
    const int pitch = RING ? ring : T;
    float acc = bu[co];
    for (int m = n / stride; m >= 0; m--) {
        const int k = n - m * stride;
        if (k >= K) break;
        if (m >= T) continue;
        const int col = RING ? m % ring : m;
        for (int ci = 0; ci < C; ci++) {
            const float w = WU_T ? Wu[((size_t)k * C + ci) * C + co] : Wu[((size_t)ci * C + co) * K + k];
            acc = fmaf(feat[((size_t)b * C + ci) * pitch + col], w, acc);
        }
    }
    return acc;
}

// y[b][o][n] of the 1x1 convolution from u stored as U[b][n][C] (channel fastest); Wc [L*2R][C]
__host__ __device__ inline float project_element(const float* __restrict__ Urow, const float* __restrict__ Wc, const float* __restrict__ bc, int C, int o)
{
    float acc = bc[o];
    const float* w = Wc + (size_t)o * C;
    for (int co = 0; co < C; co++) acc = fmaf(Urow[co], w[co], acc);
    return acc;
}

__global__ void transpose_wu_kernel(float* __restrict__ dst, const float* __restrict__ src, int C, int K)
{
    const size_t total = (size_t)C * C * K;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int co = (int)(i % C), ci = (int)((i / C) % C), k = (int)(i / ((size_t)C * C));     // dst index [k][ci][co]
        dst[i] = src[((size_t)ci * C + co) * K + k];
    }
}

// U[i][j][co] for the k rows of a chunk, row i = absolute sample n0 + j of the utterance in tab[i], i.e. sample n0 + j - start of
// its own frames [C][T] at frames + foff, or with RING its ring [C][ring] there.  Samples at or past its end (T * stride) are left
// at 0: mask_slots_kernel zeroes their projected rows.
template <bool RING>
__global__ void upsample_slots_kernel(float* __restrict__ U, const float* __restrict__ frames, const WnCondSlot* __restrict__ tab,
                                      const float* __restrict__ WuT, const float* __restrict__ bu, int k, int C, int K, int stride, long long n0, int m)
{
    const size_t total = (size_t)k * m * C;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int co = (int)(i % C), j = (int)((i / C) % m), r = (int)(i / ((size_t)C * m));
        const WnCondSlot s = tab[r];
        const long long n = n0 + j - s.start;
        U[i] = n < (long long)s.T * stride ? upsample_element<true, RING>(frames + s.foff, WuT, bu, C, s.T, K, stride, 0, co, (int)n, s.ring) : 0.f;
    }
}

// zeroes out[j][l][r][c] for every (j, r) whose sample n0 + j is at or past the end of row r's utterance (the projection of a zero
// U row is the bias, not 0).  One thread per (j, r); launched only for a chunk in which some row's utterance ends.
__global__ void mask_slots_kernel(float* __restrict__ out, const WnCondSlot* __restrict__ tab, int k, int L, int R2, int stride, long long n0, int m)
{
    const size_t total = (size_t)m * k;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int r = (int)(i % k), j = (int)(i / k);
        if (n0 + j - tab[r].start < (long long)tab[r].T * stride) continue;
        for (int l = 0; l < L; l++) {
            float* row = out + (((size_t)j * L + l) * k + r) * R2;
            for (int c = 0; c < R2; c++) row[c] = 0.f;
        }
    }
}

// out[j][l][b][c] (the engine's fp32 conditioning layout for samples n0 + j) from U[b][j][C]
__global__ void project_kernel(float* __restrict__ out, const float* __restrict__ U, const float* __restrict__ Wc, const float* __restrict__ bc,
                               int B, int C, int L, int R2, int m)
{
    const size_t total = (size_t)m * L * B * R2;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % R2), b = (int)((i / R2) % B), l = (int)((i / ((size_t)R2 * B)) % L), j = (int)(i / ((size_t)R2 * B * L));
        out[i] = project_element(U + ((size_t)b * m + j) * C, Wc, bc, C, l * R2 + c);
    }
}

// Tiled projection: rows r = j * B + b (sample-major, the order of the output), columns o = l * 2R + c; out = bc[o] + sum_co U[r][co] * Wc[o][co]
// with co ascending (project_element's order).  CTA 256 threads = 16 x 16, thread (ty, tx): rows ty*8 .. +7, columns tx*4 .. +3 and 64 + tx*4 .. +3.
constexpr int PT = 128, PK = 16;
__global__ void __launch_bounds__(256) project_tiled_kernel(float* __restrict__ out, const float* __restrict__ U, const float* __restrict__ Wc, const float* __restrict__ bc,
                                                            int B, int C, int L, int R2, int m)
{
    __shared__ __align__(16) float Us[PK][PT];
    __shared__ __align__(16) float Ws[PK][PT];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const long rows = (long)m * B;
    const int cols = L * R2;
    const long r0 = (long)blockIdx.x * PT;
    const int o0 = blockIdx.y * PT;
    // loader: thread -> (tile row lr, 8 consecutive k)
    const int lr = tid >> 1, lk = (tid & 1) * 8;
    const long ur = r0 + lr;
    const float* usrc = nullptr;
    if (ur < rows) { const long j = ur / B; const int b = (int)(ur - j * B); usrc = U + ((size_t)b * m + j) * C; }
    const int wo = o0 + lr;
    const float* wsrc = wo < cols ? Wc + (size_t)wo * C : nullptr;

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; i++) {
#pragma unroll
        for (int q = 0; q < 8; q++) { const int o = o0 + (q < 4 ? tx * 4 + q : 64 + tx * 4 + q - 4); acc[i][q] = o < cols ? bc[o] : 0.f; }
    }
    for (int k0 = 0; k0 < C; k0 += PK) {
#pragma unroll
        for (int q = 0; q < 8; q++) {
            const int k = k0 + lk + q;
            Us[lk + q][lr] = (usrc && k < C) ? usrc[k] : 0.f;
            Ws[lk + q][lr] = (wsrc && k < C) ? wsrc[k] : 0.f;
        }
        __syncthreads();
        const int kn = C - k0 < PK ? C - k0 : PK;
        for (int k = 0; k < kn; k++) {
            const float4 ua = *reinterpret_cast<const float4*>(&Us[k][ty * 8]), ub = *reinterpret_cast<const float4*>(&Us[k][ty * 8 + 4]);
            const float4 wa = *reinterpret_cast<const float4*>(&Ws[k][tx * 4]), wb = *reinterpret_cast<const float4*>(&Ws[k][64 + tx * 4]);
            const float u[8] = {ua.x, ua.y, ua.z, ua.w, ub.x, ub.y, ub.z, ub.w};
            const float w[8] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w};
#pragma unroll
            for (int i = 0; i < 8; i++) {
#pragma unroll
                for (int q = 0; q < 8; q++) acc[i][q] = fmaf(u[i], w[q], acc[i][q]);
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const long r = r0 + ty * 8 + i;
        if (r >= rows) continue;
        const long j = r / B; const int b = (int)(r - j * B);
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int o = o0 + h * 64 + tx * 4;                // four consecutive columns: same layer (4 | 2R)
            if (o >= cols) continue;
            const int l = o / R2, c = o - l * R2;
            *reinterpret_cast<float4*>(out + (((size_t)j * L + l) * B + b) * R2 + c) = make_float4(acc[i][4 * h], acc[i][4 * h + 1], acc[i][4 * h + 2], acc[i][4 * h + 3]);
        }
    }
}

unsigned grid_for(size_t total)
{
    size_t blocks = (total + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    return (unsigned)(blocks ? blocks : 1);
}

// out[j][l][b][2R] from U[b][j][C], j < m: the tiled kernel where its float4 stores fit, else the simple one
cudaError_t project(float* out, const float* U, const float* Wc, const float* bc, int B, int C, int L, int R, int m, cudaStream_t stream)
{
    const int R2 = 2 * R;
    if (R2 % 4 == 0 && (((size_t)out) & 15) == 0) {
        const dim3 grid((unsigned)(((size_t)m * B + PT - 1) / PT), (unsigned)((L * R2 + PT - 1) / PT));
        project_tiled_kernel<<<grid, 256, 0, stream>>>(out, U, Wc, bc, B, C, L, R2, m);
    } else {
        project_kernel<<<grid_for((size_t)m * L * B * R2), 256, 0, stream>>>(out, U, Wc, bc, B, C, L, R2, m);
    }
    return cudaGetLastError();
}

}  // namespace

// device pointers throughout; WuT = [K][C][C] transpose made by wn_cond_transpose_wu; U scratch holds B * m * C floats
cudaError_t wn_cond_transpose_wu(float* WuT, const float* Wu, int C, int K, cudaStream_t stream)
{
    transpose_wu_kernel<<<grid_for((size_t)C * C * K), 256, 0, stream>>>(WuT, Wu, C, K);
    return cudaGetLastError();
}

cudaError_t wn_cond_produce_slots(float* out, float* U, const float* frames, const WnCondSlot* tab, const float* WuT, const float* bu, const float* Wc,
                                  const float* bc, int k, int C, int K, int stride, int L, int R, long long n0, int m, bool mask, bool ring,
                                  cudaStream_t stream)
{
    if (m <= 0) return cudaSuccess;
    if (ring) upsample_slots_kernel<true><<<grid_for((size_t)k * m * C), 256, 0, stream>>>(U, frames, tab, WuT, bu, k, C, K, stride, n0, m);
    else upsample_slots_kernel<false><<<grid_for((size_t)k * m * C), 256, 0, stream>>>(U, frames, tab, WuT, bu, k, C, K, stride, n0, m);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = project(out, U, Wc, bc, k, C, L, R, m, stream);     // rows b * m + j -> out[j][l][b][2R]: the chunk's layout
    if (e != cudaSuccess || !mask) return e;
    mask_slots_kernel<<<grid_for((size_t)m * k), 256, 0, stream>>>(out, tab, k, L, 2 * R, stride, n0, m);
    return cudaGetLastError();
}

// Host reference of the same arithmetic (no GPU): Lh [T*stride][L][B][2R]
void wn_cond_host(float* Lh, const float* feat, const float* Wu, const float* bu, const float* Wc, const float* bc,
                  int B, int C, int T, int K, int stride, int L, int R)
{
    const int Nn = T * stride, R2 = 2 * R;
    float* Urow = new float[C];
    for (int b = 0; b < B; b++)
        for (int n = 0; n < Nn; n++) {
            for (int co = 0; co < C; co++) Urow[co] = upsample_element<false>(feat, Wu, bu, C, T, K, stride, b, co, n);
            for (int l = 0; l < L; l++)
                for (int c = 0; c < R2; c++)
                    Lh[(((size_t)n * L + l) * B + b) * R2 + c] = project_element(Urow, Wc, bc, C, l * R2 + c);
        }
    delete[] Urow;
}
