// wn_convert.cu -- dtype conversion / fill helpers (replaces nv_wavenet_conversions.cuh:28-116).
#include "wn_common.h"

namespace {
__global__ void f32_to_f16_kernel(__half* __restrict__ dst, const float* __restrict__ src, size_t n)
{
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    // 4 elements per thread per trip when aligned
    const size_t n4 = ((reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst) & 7) == 0) ? n / 4 : 0;
    for (size_t j = i; j < n4; j += stride) {
        const float4 v = reinterpret_cast<const float4*>(src)[j];
        __half2 lo = __floats2half2_rn(v.x, v.y), hi = __floats2half2_rn(v.z, v.w);
        uint2 o;
        o.x = *reinterpret_cast<unsigned*>(&lo);
        o.y = *reinterpret_cast<unsigned*>(&hi);
        reinterpret_cast<uint2*>(dst)[j] = o;
    }
    for (size_t j = n4 * 4 + i; j < n; j += stride) dst[j] = __float2half_rn(src[j]);
}
// mu-law decode of sampled indices, table-driven: out[b][j] = lut[yOut[b * N + offset + j]]
__global__ void mulaw_decode_kernel(const int* __restrict__ y, int N, int offset, int size, size_t total, int A, const float* __restrict__ lut_f,
                                    const short* __restrict__ lut_s, float* __restrict__ out_f, short* __restrict__ out_s)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t b = i / (size_t)size, j = i % (size_t)size;
        int v = y[b * (size_t)N + offset + j];
        v = v < 0 ? 0 : (v >= A ? A - 1 : v);
        if (out_f) out_f[i] = lut_f[v];
        if (out_s) out_s[i] = lut_s[v];
    }
}
__global__ void fill_int_kernel(int* dst, int v, size_t n)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] = v;
}
}  // namespace

cudaError_t wn_f32_to_f16(__half* dst, const float* src_dev, size_t n, cudaStream_t stream)
{
    if (n == 0) return cudaSuccess;
    const int threads = 256;
    size_t blocks = (n / 4 + threads - 1) / threads;
    if (blocks < 1) blocks = 1;
    if (blocks > 132 * 16) blocks = 132 * 16;
    f32_to_f16_kernel<<<(unsigned)blocks, threads, 0, stream>>>(dst, src_dev, n);
    return cudaGetLastError();
}

__global__ void f16_to_f32_kernel(float* __restrict__ dst, const __half* __restrict__ src, size_t n)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] = __half2float(src[i]);
}
cudaError_t wn_f16_to_f32(float* dst, const __half* src_dev, size_t n, cudaStream_t stream)
{
    if (n == 0) return cudaSuccess;
    size_t blocks = (n + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    f16_to_f32_kernel<<<(unsigned)blocks, 256, 0, stream>>>(dst, src_dev, n);
    return cudaGetLastError();
}

// Counter-based selectors (SURVEY.md 8f next-1: "device-side Philox selectors"): element i of the [N][B] selector array is the
// first 32-bit output of Philox-4x32-10 with counter (i_lo, i_hi, 0, 0) and key (seed_lo, seed_hi), mapped to [0, 1) with
// 24 bits: (x >> 8) * 2^-24.  Stateless, order-independent, reproducible on the host (tests/test_gpu_zz_selectors.py).
__host__ __device__ inline unsigned wn_philox_first(unsigned long long ctr, unsigned long long seed)
{
    unsigned c0 = (unsigned)ctr, c1 = (unsigned)(ctr >> 32), c2 = 0, c3 = 0;
    unsigned k0 = (unsigned)seed, k1 = (unsigned)(seed >> 32);
    for (int r = 0; r < 10; r++) {
        const unsigned long long p0 = (unsigned long long)0xD2511F53u * c0, p1 = (unsigned long long)0xCD9E8D57u * c2;
        const unsigned n0 = (unsigned)(p1 >> 32) ^ c1 ^ k0, n1 = (unsigned)p1, n2 = (unsigned)(p0 >> 32) ^ c3 ^ k1, n3 = (unsigned)p0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    return c0;
}
__global__ void selectors_kernel(float* __restrict__ dst, size_t n, unsigned long long seed, unsigned long long first)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        dst[i] = (float)(wn_philox_first(first + i, seed) >> 8) * (1.0f / 16777216.0f);
}
// dst[i] = selector of counter first + i
cudaError_t wn_fill_selectors(float* dst, size_t n, unsigned long long seed, unsigned long long first, cudaStream_t stream)
{
    if (n == 0) return cudaSuccess;
    size_t blocks = (n + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    selectors_kernel<<<(unsigned)blocks, 256, 0, stream>>>(dst, n, seed, first);
    return cudaGetLastError();
}

// Per-slot selectors (continuous batching): slot b at absolute sample t draws counter t - origin[b] under key seed[b], which is
// what a one-utterance engine draws at sample t - origin[b] (counter sample * 1 + 0): an utterance's selectors do not depend on
// its slot, its start time or the batch it shares.
__global__ void selectors_slots_kernel(float* __restrict__ dst, size_t n, int B, long long first_t, const long long* __restrict__ origin,
                                       const unsigned long long* __restrict__ seed)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int b = (int)(i % B);
        const long long t = first_t + (long long)(i / B);
        dst[i] = (float)(wn_philox_first((unsigned long long)(t - origin[b]), seed[b]) >> 8) * (1.0f / 16777216.0f);
    }
}
cudaError_t wn_fill_selectors_slots(float* dst, int n, int B, long long first_t, const long long* origin, const unsigned long long* seed,
                                    cudaStream_t stream)
{
    const size_t total = (size_t)n * B;
    if (total == 0) return cudaSuccess;
    size_t blocks = (total + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    selectors_slots_kernel<<<(unsigned)blocks, 256, 0, stream>>>(dst, total, B, first_t, origin, seed);
    return cudaGetLastError();
}

__global__ void restart_rows_kernel(const int* __restrict__ rows, int n, const unsigned long long* __restrict__ seeds, long long t0,
                                    int* yPrev, int* yCur, long long* origin, unsigned long long* seed)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int b = rows[i];
        yPrev[b] = 128;                   // silence, as nvwn_reset_history
        yCur[b] = 128;
        origin[b] = t0;
        seed[b] = seeds ? seeds[i] : 0ull;
    }
}
cudaError_t wn_restart_rows(const int* rows, int n, const unsigned long long* seeds, long long t0, int* yPrev, int* yCur, long long* origin,
                            unsigned long long* seed, cudaStream_t stream)
{
    if (n <= 0) return cudaSuccess;
    restart_rows_kernel<<<(n + 255) / 256, 256, 0, stream>>>(rows, n, seeds, t0, yPrev, yCur, origin, seed);
    return cudaGetLastError();
}

cudaError_t wn_fill_int(int* dst, int value, size_t n, cudaStream_t stream)
{
    if (n == 0) return cudaSuccess;
    size_t blocks = (n + 255) / 256;
    if (blocks > 1024) blocks = 1024;
    fill_int_kernel<<<(unsigned)blocks, 256, 0, stream>>>(dst, value, n);
    return cudaGetLastError();
}

cudaError_t wn_plain_convert(const WnConfig& c, void* store, const float* src, int first_sample, int num_samples, cudaStream_t stream)
{
    const size_t per = (size_t)c.L * c.B * 2 * c.R, n = per * num_samples;
    if (c.dtype == NVWN_FP16) return wn_f32_to_f16(static_cast<__half*>(store) + (size_t)first_sample * per, src, n, stream);
    return cudaMemcpyAsync(static_cast<float*>(store) + (size_t)first_sample * per, src, n * sizeof(float), cudaMemcpyDefault, stream);
}

cudaError_t wn_plain_readback(const WnConfig& c, float* dst_dev, const void* store, int first_sample, int num_samples, cudaStream_t stream)
{
    const size_t per = (size_t)c.L * c.B * 2 * c.R, n = per * num_samples;
    if (c.dtype == NVWN_FP16) return wn_f16_to_f32(dst_dev, static_cast<const __half*>(store) + (size_t)first_sample * per, n, stream);
    return cudaMemcpyAsync(dst_dev, static_cast<const float*>(store) + (size_t)first_sample * per, n * sizeof(float), cudaMemcpyDeviceToDevice, stream);
}

// fed-back indices from the codes of a scoring stream: step t embeds (y[t-2], y[t-1]) = (yPrev, yCur) in generation and
// (codes[b][0], codes[b][1]) at the first step of the scorer's next call
__global__ void feedback_from_codes_kernel(const int* __restrict__ codes, int n, int* yPrev, int* yCur)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < n) {
        yPrev[b] = codes[2 * b];
        yCur[b] = codes[2 * b + 1];
    }
}
cudaError_t wn_feedback_from_codes(const int* codes, int n, int* yPrev, int* yCur, cudaStream_t stream)
{
    if (n <= 0) return cudaSuccess;
    feedback_from_codes_kernel<<<(n + 255) / 256, 256, 0, stream>>>(codes, n, yPrev, yCur);
    return cudaGetLastError();
}

// the per-slot prime's state: restart_rows_kernel with the fed-back indices of feedback_from_codes_kernel
__global__ void prime_rows_kernel(const int* __restrict__ codes, const int* __restrict__ rows, const int* __restrict__ slots, int n,
                                  const unsigned long long* __restrict__ seeds, long long t_origin, int* yPrev, int* yCur, long long* origin,
                                  unsigned long long* seed)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int b = slots[i], r = rows[i];
        yPrev[b] = codes[2 * r];
        yCur[b] = codes[2 * r + 1];
        origin[b] = t_origin;
        seed[b] = seeds ? seeds[i] : 0ull;
    }
}
cudaError_t wn_prime_rows(const int* codes, const int* rows, const int* slots, int n, const unsigned long long* seeds, long long t_origin, int* yPrev,
                          int* yCur, long long* origin, unsigned long long* seed, cudaStream_t stream)
{
    if (n <= 0) return cudaSuccess;
    prime_rows_kernel<<<(n + 255) / 256, 256, 0, stream>>>(codes, rows, slots, n, seeds, t_origin, yPrev, yCur, origin, seed);
    return cudaGetLastError();
}

// the header, then per layer its d_l history rows of R elements of the ring's type
size_t wn_slot_state_bytes(const WnConfig& c)
{
    size_t rows = 0;
    for (int l = 0; l < c.L; l++) rows += (size_t)wn_score_dilation(l, c.maxDil);
    return sizeof(nvwn_slot_state_header) + rows * c.R * (c.dtype == NVWN_FP16 ? sizeof(__half) : sizeof(float));
}

// Slot states (DESIGN.md §6): the scalar fields, next to the history rows the layout kernels move.  The position is computed here
// from the slot's origin, so a save needs no host synchronisation.
__global__ void save_slot_scalars_kernel(char* states, size_t bytes, const int* __restrict__ rows, int n, nvwn_slot_state_header h, long long next_t,
                                         const int* __restrict__ yPrev, const int* __restrict__ yCur, const long long* __restrict__ origin,
                                         const unsigned long long* __restrict__ seed)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int b = rows[i];
        h.y_prev = yPrev[b];
        h.y_cur = yCur[b];
        h.position = next_t - origin[b];
        h.seed = seed[b];
        *reinterpret_cast<nvwn_slot_state_header*>(states + (size_t)i * bytes) = h;
    }
}
cudaError_t wn_save_slot_scalars(void* states, size_t bytes, const int* rows, int n, const WnConfig& c, long long next_t, const int* yPrev,
                                 const int* yCur, const long long* origin, const unsigned long long* seed, cudaStream_t stream)
{
    if (n <= 0) return cudaSuccess;
    nvwn_slot_state_header h = {};
    h.tag = NVWN_SLOT_STATE_TAG;
    h.dtype = c.dtype; h.R = c.R; h.L = c.L; h.max_dilation = c.maxDil;
    save_slot_scalars_kernel<<<(n + 255) / 256, 256, 0, stream>>>(static_cast<char*>(states), bytes, rows, n, h, next_t, yPrev, yCur, origin, seed);
    return cudaGetLastError();
}

// Slot states of scoring rows (nvwn_score_save_states): block (x, i) writes parts of state i.  Its body is the concatenation over
// layers of the fronts' rows of scoring row rows[i], [d_l][R] fp16 each, moved as 16-byte vectors; row g of the body is layer l's
// front row g - (d_0 + .. + d_{l-1}), which sits at xh + wn_score_xh_offset(l) time-major [d_l][Bs][R] (the layers' buffers are
// [d_l + Tcap][Be][R] apart, the rows inside at the scoring stream's batch Bs).  Block (0, i) also writes the
// header: position P, the row's codes of steps P - 2 and P - 1, seeds[i] (seeds NULL: 0).
__global__ void score_save_states_kernel(char* states, size_t bytes, const __half* __restrict__ xh, const int* __restrict__ codes,
                                         const int* __restrict__ rows, const unsigned long long* __restrict__ seeds, nvwn_slot_state_header h,
                                         int L, int R, int maxDil, int Tcap, int Be, int Bs, size_t vecs)
{
    const int i = blockIdx.y, row = rows[i];
    char* st = states + (size_t)i * bytes;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        h.y_prev = codes[2 * row];
        h.y_cur = codes[2 * row + 1];
        h.seed = seeds ? seeds[i] : 0ull;
        *reinterpret_cast<nvwn_slot_state_header*>(st) = h;
    }
    const int vpr = R * (int)sizeof(__half) / 16;                       // vectors per [R] row
    uint4* body = reinterpret_cast<uint4*>(st + sizeof(nvwn_slot_state_header));
    for (size_t v = (size_t)blockIdx.x * blockDim.x + threadIdx.x; v < vecs; v += (size_t)gridDim.x * blockDim.x) {
        const int g = (int)(v / vpr), c = (int)(v % vpr);
        int first = 0, d = 1;                                           // layer l's first body row and d_l
        size_t off = 0;                                                 // wn_score_xh_offset(l)
        for (int l = 0; l < L && g >= first + d; l++) {
            off += ((size_t)d + Tcap) * Be * R;
            first += d;
            d = 2 * d > maxDil ? 1 : 2 * d;
        }
        body[v] = reinterpret_cast<const uint4*>(xh + off + ((size_t)(g - first) * Bs + row) * R)[c];
    }
}
cudaError_t wn_score_save_states(void* states, size_t bytes, const __half* xh, const int* codes, const int* rows, int n, const unsigned long long* seeds,
                                 const WnConfig& c, long long P, int Tcap, int Be, int Bs, cudaStream_t stream)
{
    if (n <= 0) return cudaSuccess;
    nvwn_slot_state_header h = {};
    h.tag = NVWN_SLOT_STATE_TAG;
    h.dtype = NVWN_FP16; h.R = c.R; h.L = c.L; h.max_dilation = c.maxDil;
    h.position = P;
    const size_t vecs = (bytes - sizeof(nvwn_slot_state_header)) / 16;
    const unsigned blocks = (unsigned)((vecs + 255) / 256 < 64 ? (vecs + 255) / 256 : 64);
    score_save_states_kernel<<<dim3(blocks, (unsigned)n), 256, 0, stream>>>(static_cast<char*>(states), bytes, xh, codes, rows, seeds, h, c.L, c.R,
                                                                            c.maxDil, Tcap, Be, Bs, vecs);
    return cudaGetLastError();
}

__global__ void load_slot_scalars_kernel(const char* states, size_t bytes, const int* __restrict__ rows, int n, long long t0, int* yPrev, int* yCur,
                                         long long* origin, unsigned long long* seed)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int b = rows[i];
        const nvwn_slot_state_header h = *reinterpret_cast<const nvwn_slot_state_header*>(states + (size_t)i * bytes);
        yPrev[b] = h.y_prev;
        yCur[b] = h.y_cur;
        origin[b] = t0 - h.position;
        seed[b] = h.seed;
    }
}
cudaError_t wn_load_slot_scalars(const void* states, size_t bytes, const int* rows, int n, long long t0, int* yPrev, int* yCur, long long* origin,
                                 unsigned long long* seed, cudaStream_t stream)
{
    if (n <= 0) return cudaSuccess;
    load_slot_scalars_kernel<<<(n + 255) / 256, 256, 0, stream>>>(static_cast<const char*>(states), bytes, rows, n, t0, yPrev, yCur, origin, seed);
    return cudaGetLastError();
}

cudaError_t wn_mulaw_decode(const int* yOut, int N, int offset, int size, int B, int A, const float* lut_f, const short* lut_s, float* out_f,
                            short* out_s, cudaStream_t stream)
{
    const size_t total = (size_t)B * size;
    if (total == 0) return cudaSuccess;
    size_t blocks = (total + 255) / 256;
    if (blocks > 132 * 8) blocks = 132 * 8;
    mulaw_decode_kernel<<<(unsigned)blocks, 256, 0, stream>>>(yOut, N, offset, size, total, A, lut_f, lut_s, out_f, out_s);
    return cudaGetLastError();
}
