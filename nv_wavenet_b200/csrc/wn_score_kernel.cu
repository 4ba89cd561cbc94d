// wn_score_kernel.cu -- teacher-forced scoring: log p(audio[b][t] | audio[b][0..t), conditioning) for every step at once
// (nvwn_score, DESIGN.md §5.4).
//
// With the audio given, step t no longer waits for step t-1, so the rows m = (t, b) of a time chunk are independent and every
// per-sample matrix-vector product of generation becomes one GEMM over T * Bs rows:
//   embed   x_0 = [tanh](embPrev[a[t-2]] + embCur[a[t-1]])                                 (one launch)
//   layer l a = [x_l[t] | x_l[t-d]] . [Wcur_l | Wprev_l]^T + Bh_l + Lh[t][l]  (K = 2R)
//           h = tanh(a[:R]) * sigmoid(a[R:])  -> H[:, l*R : (l+1)*R]   (fp16)
//           x_{l+1} = h . Wres_l^T + Bres_l + x_l                              (fp32)       (one launch per layer)
//   output  skip = relu(H . [Wskip_0 .. Wskip_{L-1}]^T + sum Bskip)   (K = L * R)
//           Zs = relu(skip . Wzs^T + Bzs);  Za = Zs . Wza^T + Bza;  logp = Za[a[t]] - logsumexp(Za)      (one launch)
//
// Each layer's fp16 input buffer carries the last d_l steps of the previous chunk in front of the chunk, so x_l[t-d] is the
// same buffer d_l * Bs rows earlier.  A scoring stream (nvwn_score_stream) keeps those fronts and the last two codes between
// calls, so the first chunk of a call continues the previous call's last one.  Tensor cores through mma.sync.m16n8k16 (fp16 in,
// fp32 accumulate) from XOR-swizzled shared-memory tiles loaded with cp.async; every output element accumulates its K in one
// fixed order in one CTA (no split-K, no atomics), so a row's result does not depend on which tile, chunk or batch it is computed in.
// Packed scoring (nvwn_score_stream_packed) starts utterances inside a row: the PACKED instantiations of the embedding and layer
// kernels read codes 128 and zero x[t-d] by each row's local time, where a fresh start reads the 128s and the zeroed fronts.
// Scoring by model (nvwn_set_score_models): the MODELS instantiations take the chunk's rows model by model (WnScoreSegs), in tiles
// of one model each, and read each tile's weights from its model's image; a row's arithmetic is the one-model kernels', so its
// results are the bits an engine holding its model as model 0 gives.
#include "wn_common.h"
#include "wn_math.cuh"

namespace {

constexpr int BM = 64;                 // rows per tile
constexpr int NTHREADS = 256;          // 8 warps: 4 along the rows (16 each) x 2 along the columns
constexpr int KS = 64;                 // k-slice of the streamed GEMMs of the output kernel
constexpr int A_OUT = 256;             // output channels the output kernel is built for

struct ImageLayout {
    size_t W1, Wr, Ws, Wzs, Wza, Bh, Br, Bsk, Bzs, Bza, bytes;
};

ImageLayout image_layout(int R, int S, int A, int L)
{
    ImageLayout o;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t r = off; off = (off + bytes + 255) / 256 * 256; return r; };
    o.W1 = take((size_t)L * 4 * R * R * 2);          // per layer [2R][2R]: row n = output channel, k < R from Wcur, k >= R from Wprev
    o.Wr = take((size_t)L * R * R * 2);              // per layer [R][R]
    o.Ws = take((size_t)S * L * R * 2);              // [S][L*R]
    o.Wzs = take((size_t)A * S * 2);                 // [A][S]
    o.Wza = take((size_t)A * A * 2);                 // [A][A]
    o.Bh = take((size_t)L * 2 * R * 4);              // fp32 biases
    o.Br = take((size_t)L * R * 4);
    o.Bsk = take((size_t)S * 4);                     // sum over the layers of Bskip
    o.Bzs = take((size_t)A * 4);
    o.Bza = take((size_t)A * 4);
    o.bytes = off;
    return o;
}

// ---- packing: engine blob (fp16, column-major M x K, W[row + k * M]) -> k-contiguous rows ----
__global__ void pack_w1_kernel(__half* __restrict__ out, const __half* __restrict__ Wcur, const __half* __restrict__ Wprev, int R, int L)
{
    const size_t n_all = (size_t)L * 4 * R * R;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_all; i += (size_t)gridDim.x * blockDim.x) {
        const size_t l = i / (4 * R * R);
        const int n = (int)(i / (2 * R) % (2 * R)), k = (int)(i % (2 * R));
        const __half* W = (k < R ? Wcur : Wprev) + l * 2 * R * R;
        out[i] = W[n + (size_t)(k % R) * 2 * R];
    }
}
// out[(b * M + n) * ld_out... ]: batch `nb` of column-major M x K matrices (stride in_stride) -> rows of K at out + b * out_off + n * ld
__global__ void pack_t_kernel(__half* __restrict__ out, size_t out_off, int ld, const __half* __restrict__ W, size_t in_stride, int M, int K, int nb)
{
    const size_t n_all = (size_t)nb * M * K;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_all; i += (size_t)gridDim.x * blockDim.x) {
        const size_t b = i / ((size_t)M * K);
        const int n = (int)(i / K % M), k = (int)(i % K);
        out[b * out_off + (size_t)n * ld + k] = W[b * in_stride + n + (size_t)k * M];
    }
}
__global__ void pack_bias_kernel(float* __restrict__ Bh, float* __restrict__ Br, float* __restrict__ Bsk, float* __restrict__ Bzs, float* __restrict__ Bza,
                                 const __half* __restrict__ bh, const __half* __restrict__ br, const __half* __restrict__ bsk, const __half* __restrict__ bzs,
                                 const __half* __restrict__ bza, int R, int S, int A, int L)
{
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nt = gridDim.x * blockDim.x;
    for (int i = tid; i < L * 2 * R; i += nt) Bh[i] = __half2float(bh[i]);
    for (int i = tid; i < L * R; i += nt) Br[i] = __half2float(br[i]);
    for (int s = tid; s < S; s += nt) {
        float v = 0.f;
        for (int l = 0; l < L; l++) v += __half2float(bsk[(size_t)l * S + s]);
        Bsk[s] = v;
    }
    for (int a = tid; a < A; a += nt) { Bzs[a] = __half2float(bzs[a]); Bza[a] = __half2float(bza[a]); }
}

// the codes of the next call's steps -2 and -1: the last two of this call's `count` codes (row stride N); with count = 1 the
// pair shifts by one
__global__ void carry_codes_kernel(int* __restrict__ codes, const int* __restrict__ audio, int N, int count, int Bs)
{
    for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < Bs; b += gridDim.x * blockDim.x) {
        const int prev = count >= 2 ? audio[(size_t)b * N + count - 2] : codes[2 * b + 1];
        codes[2 * b] = prev;
        codes[2 * b + 1] = audio[(size_t)b * N + count - 1];
    }
}

__global__ void check_audio_kernel(const int* __restrict__ audio, size_t n, int A, unsigned long long* first_bad)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int v = audio[i];
        if (v < 0 || v >= A) atomicMin(first_bad, (unsigned long long)i);
    }
}

// ---- tensor-core helpers ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// byte offset of 16-byte chunk c of row r in a tile of nch chunks per row; chunks XOR-swizzled so ldmatrix is conflict-free
__device__ __forceinline__ uint32_t swz(int r, int c, int nch)
{
    const int m = (nch < 8 ? nch : 8) - 1;
    return (uint32_t)(r * nch + (c ^ (r & m))) * 16u;
}
__device__ __forceinline__ void cp16(uint32_t dst, const void* src, bool valid)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0));
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N> __device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }
__device__ __forceinline__ void ldsm4(uint32_t (&r)[4], uint32_t addr)
{
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
{
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// A fragment: rows r0..r0+15, k chunks kc, kc+1 of a row-major tile
__device__ __forceinline__ void load_a(uint32_t (&a)[4], uint32_t base, int nch, int r0, int kc, int lane)
{
    ldsm4(a, base + swz(r0 + (lane & 15), kc + (lane >> 4), nch));
}
// B fragments of two n-tiles (columns n0..n0+15), k chunks kc, kc+1, of a [N][K] tile: {b0, b1} of n0, {b0, b1} of n0+8
__device__ __forceinline__ void load_b2(uint32_t (&b)[4], uint32_t base, int nch, int n0, int kc, int lane)
{
    ldsm4(b, base + swz(n0 + (lane & 7) + ((lane >> 4) << 3), kc + ((lane >> 3) & 1), nch));
}
__device__ __forceinline__ void sts32(uint32_t addr, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;\n" ::"r"(addr), "r"(v)); }
__device__ __forceinline__ uint32_t u32(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }

// ---- embedding: x_0 of every row of the chunk; the codes of call steps -2 and -1 come from codes[b][0..1] ----
// PACKED (nvwn_score_stream_packed): tau[m] is row m's local time, the samples its utterance has run before this one; the codes of
// its steps -1 and -2 are 128 where tau < 1 and tau < 2
// MODELS: row b reads the embeddings of its model segs->row_model[b]
template <bool PACKED, bool MODELS>
__global__ void score_embed_kernel(const __half* __restrict__ embPrev, const __half* __restrict__ embCur, const int* __restrict__ audio,
                                   const int* __restrict__ codes, int N, int t0, int M, int Bs, int R, int tanhEmbed, float* __restrict__ xf,
                                   __half* __restrict__ x0, const int* __restrict__ tau, const WnScoreSegs* __restrict__ segs)
{
    const size_t n_all = (size_t)M * R;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_all; i += (size_t)gridDim.x * blockDim.x) {
        const int m = (int)(i / R), r = (int)(i % R), b = m % Bs, t = t0 + m / Bs;
        int yp = t >= 2 ? audio[(size_t)b * N + t - 2] : codes[2 * b + t], yc = t >= 1 ? audio[(size_t)b * N + t - 1] : codes[2 * b + 1];
        if (PACKED) {
            const int tm = tau[m];
            if (tm < 2) yp = 128;
            if (tm < 1) yc = 128;
        }
        const __half *eP = embPrev, *eC = embCur;
        if (MODELS) {
            const int v = segs->row_model[b];
            eP = static_cast<const __half*>(segs->embPrev[v]);
            eC = static_cast<const __half*>(segs->embCur[v]);
        }
        float v = __half2float(eP[(size_t)yp * R + r]) + __half2float(eC[(size_t)yc * R + r]);
        if (tanhEmbed) v = wn::tanhf_fast(v);         // as the latency kernel (wn_lat_kernel.cu)
        xf[i] = v;
        x0[i] = __float2half_rn(v);
    }
}

// ---- packed scoring: tau [T][Bs] of the chunk's rows from the call's start flags [Bs][N]; carry[b] is the tau row b's next sample
// has without a flag (0 when a stream opens), and leaves as that of the sample after the chunk.  Clamped at cap = max(maxDil, 2):
// the kernels only compare tau with 1, 2 and d_l <= maxDil.  One warp per row, 32 steps at a time: a lane's tau counts from the
// last flag at or before it, or on from the carry ----
__global__ void score_tau_kernel(int* __restrict__ tau, int* __restrict__ carry, const unsigned char* __restrict__ starts, int N, int t0, int T,
                                 int Bs, int cap)
{
    const int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (b >= Bs) return;                              // whole warps
    int c = carry[b];
    for (int i0 = 0; i0 < T; i0 += 32) {
        const int i = i0 + lane;
        const bool f = i < T && starts[(size_t)b * N + t0 + i];
        const unsigned m = __ballot_sync(0xffffffffu, f) & (0xffffffffu >> (31 - lane));     // flags at lanes <= lane
        int v = m ? lane - (31 - __clz(m)) : c + lane;
        v = v < cap ? v : cap;
        if (i < T) tau[(size_t)i * Bs + b] = v;
        const int last = __shfl_sync(0xffffffffu, v, T - 1 - i0 < 31 ? T - 1 - i0 : 31);
        c = last + 1 < cap ? last + 1 : cap;
    }
    if (lane == 0) carry[b] = c;
}

// ---- one residual layer over all rows of the chunk; weights resident in shared memory, persistent over row tiles ----
struct LayerArgs {
    const __half *W1, *Wr;          // [2R][2R], [R][R]
    const float *Bh, *Br;           // [2R], [R]
    const __half* xin;              // layer input buffer: history rows [0, hist), chunk row m at hist + m; x[t-d] of row m is row m
    int hist;
    float* xf;                      // fp32 residual stream [M][R] (read, then overwritten with x_{l+1})
    __half* xout;                   // next layer's chunk rows (x_{l+1} in fp16), NULL for the last layer
    __half* H;                      // gate output at column l * R, row stride ldh
    int ldh;
    const float* lh;                // conditioning of this layer: row (tl, b) at lh + tl * lh_t + b * 2R
    size_t lh_t;
    int M, Bs;
    int d;                          // the layer's dilation
    const int* tau;                 // PACKED: local time of row m (score_tau_kernel); x[t-d] reads 0 where tau[m] < d
};

// The second argument of the layer and output kernels, read by their MODELS instantiations only: the chunk's segments (device),
// their tiles, and the byte offsets in every image of the weights the launch reads (the layer's W1, Wr, Bh, Br; the output's)
struct ModelArgs {
    const WnScoreSegs* segs;
    int tiles;
    size_t oW1, oWr, oBh, oBr, oWs, oWzs, oWza, oBsk, oBzs, oBza;
};

template <int R>
__host__ __device__ constexpr int layer_smem() { return (4 * R * R + R * R + BM * 2 * R + BM * R) * 2; }

// MODELS: the segment of tile `tile` of a chunk of T steps, and in `start` the chunk tile its segment begins at
__device__ __forceinline__ int score_seg(const WnScoreSegs* __restrict__ s, int T, int tile, int& start)
{
    int k = 0, base = 0;
    for (; k + 1 < s->count; k++) {
        const int nt = (T * s->n[k] + BM - 1) / BM;
        if (tile < base + nt) break;
        base += nt;
    }
    start = base;
    return k;
}
// MODELS: the chunk row of local row q of segment k (T steps, Bs rows per step), -1 past the segment's rows
__device__ __forceinline__ int score_row(const WnScoreSegs* __restrict__ s, int k, int q, int T, int Bs)
{
    const int n = s->n[k];
    return q < T * n ? (q / n) * Bs + s->order[s->first[k] + q % n] : -1;
}

// MODELS: a CTA takes a contiguous range of the chunk's tiles (segment by segment) and loads a tile's model's weights only where
// they differ from the last tile's, so it reloads them at most once per segment boundary in its range; srow holds the chunk row of
// each of the tile's rows (-1 past its segment's rows), through which every row access goes
template <int R, bool PACKED, bool MODELS>
__global__ void __launch_bounds__(NTHREADS) score_layer_kernel(const LayerArgs a, const ModelArgs x)
{
    extern __shared__ __align__(128) unsigned char smem[];
    constexpr int N1 = 2 * R / 8, NR = R / 8, NJ = R / 16;       // chunks per row of W1 / XA, of Wr / HT; n-tiles per warp and half
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp & 3, wn = warp >> 2, g = lane >> 2, q = lane & 3;
    const uint32_t sW1 = smem_u32(smem), sWr = sW1 + 4 * R * R * 2, sXA = sWr + R * R * 2, sHT = sXA + BM * 2 * R * 2;
    int* srow = reinterpret_cast<int*>(smem + layer_smem<R>());
    const float *Bh = nullptr, *Br = nullptr;         // MODELS: the resident model's biases

    if (!MODELS) {
        for (int i = tid; i < 2 * R * N1; i += NTHREADS) cp16(sW1 + swz(i / N1, i % N1, N1), a.W1 + (size_t)i * 8, true);
        for (int i = tid; i < R * NR; i += NTHREADS) cp16(sWr + swz(i / NR, i % NR, NR), a.Wr + (size_t)i * 8, true);
        cp_commit();
    }

    const int tiles = MODELS ? x.tiles : (a.M + BM - 1) / BM;
    const int lo = MODELS ? (int)((long long)blockIdx.x * tiles / gridDim.x) : (int)blockIdx.x;
    const int hi = MODELS ? (int)((long long)(blockIdx.x + 1) * tiles / gridDim.x) : tiles;
    int resident = -1;
    for (int tile = lo; tile < hi; tile += MODELS ? 1 : gridDim.x) {
        const int m0 = tile * BM;
        if (MODELS) {
            const int T = a.M / a.Bs;
            int start;
            const int k = score_seg(x.segs, T, tile, start);
            __syncthreads();                            // the last tile's reads of srow and of the weights are done
            if (k != resident) {
                const char* im = static_cast<const char*>(x.segs->image[x.segs->model[k]]);
                const __half* W1 = reinterpret_cast<const __half*>(im + x.oW1);
                const __half* Wr = reinterpret_cast<const __half*>(im + x.oWr);
                Bh = reinterpret_cast<const float*>(im + x.oBh);
                Br = reinterpret_cast<const float*>(im + x.oBr);
                for (int i = tid; i < 2 * R * N1; i += NTHREADS) cp16(sW1 + swz(i / N1, i % N1, N1), W1 + (size_t)i * 8, true);
                for (int i = tid; i < R * NR; i += NTHREADS) cp16(sWr + swz(i / NR, i % NR, NR), Wr + (size_t)i * 8, true);
                resident = k;
            }
            if (tid < BM) srow[tid] = score_row(x.segs, k, (tile - start) * BM + tid, T, a.Bs);
            __syncthreads();
        }
        for (int i = tid; i < BM * N1; i += NTHREADS) {
            const int r = i / N1, c = i % N1, m = MODELS ? srow[r] : m0 + r;
            const bool v = MODELS ? m >= 0 : m < a.M;
            const size_t row = v ? (size_t)m + (c < NR ? a.hist : 0) : 0;
            // packed: x[t-d] of a row whose utterance began less than d samples ago is the zero a fresh start reads from its front
            cp16(sXA + swz(r, c, N1), a.xin + row * R + (c % NR) * 8, PACKED ? v && (c < NR || a.tau[m] >= a.d) : v);
        }
        cp_commit();
        cp_wait<0>();
        __syncthreads();

        // a = [x | x[t-d]] . [Wcur | Wprev]^T: this warp's tanh columns wn*R/2 + [0, R/2) and the matching sigmoid columns
        float at[NJ][4], as[NJ][4];
#pragma unroll
        for (int j = 0; j < NJ; j++)
#pragma unroll
            for (int i = 0; i < 4; i++) at[j][i] = as[j][i] = 0.f;
#pragma unroll
        for (int kk = 0; kk < 2 * R / 16; kk++) {
            uint32_t af[4];
            load_a(af, sXA, N1, wm * 16, 2 * kk, lane);
#pragma unroll
            for (int jj = 0; jj < NJ / 2; jj++) {
                uint32_t b[4];
                load_b2(b, sW1, N1, wn * (R / 2) + 16 * jj, 2 * kk, lane);
                mma(at[2 * jj], af, b[0], b[1]);
                mma(at[2 * jj + 1], af, b[2], b[3]);
                load_b2(b, sW1, N1, R + wn * (R / 2) + 16 * jj, 2 * kk, lane);
                mma(as[2 * jj], af, b[0], b[1]);
                mma(as[2 * jj + 1], af, b[2], b[3]);
            }
        }
        // + Bh + Lh, gate in the latency kernel's arithmetic: fp16 tanh.approx on the rounded pre-activations,
        // sigmoid(x) = 0.5 tanh(x / 2) + 0.5, product in fp16
        const __half2 half = __floats2half2_rn(0.5f, 0.5f);
#pragma unroll
        for (int hr = 0; hr < 2; hr++) {
            const int r = wm * 16 + g + 8 * hr, m = MODELS ? srow[r] : m0 + r;
            const bool v = MODELS ? m >= 0 : m < a.M;
            const float* lh = a.lh + (v ? (size_t)(m / a.Bs) * a.lh_t + (size_t)(m % a.Bs) * 2 * R : 0);
#pragma unroll
            for (int j = 0; j < NJ; j++) {
                const int c = wn * (R / 2) + 8 * j + 2 * q;
                const float2 bt = *reinterpret_cast<const float2*>(MODELS ? Bh + c : a.Bh + c), bs = *reinterpret_cast<const float2*>(MODELS ? Bh + R + c : a.Bh + R + c);
                float2 lt = make_float2(0.f, 0.f), ls = lt;
                if (v) { lt = *reinterpret_cast<const float2*>(lh + c); ls = *reinterpret_cast<const float2*>(lh + R + c); }
                const float t0 = (at[j][2 * hr] + bt.x) + lt.x, t1 = (at[j][2 * hr + 1] + bt.y) + lt.y;
                const float s0 = (as[j][2 * hr] + bs.x) + ls.x, s1 = (as[j][2 * hr + 1] + bs.y) + ls.y;
                const __half2 tg = wn::tanh_h2(__floats2half2_rn(t0, t1));
                const __half2 sg = __hfma2(wn::tanh_h2(__floats2half2_rn(0.5f * s0, 0.5f * s1)), half, half);
                const __half2 h = __hmul2(tg, sg);
                sts32(sHT + swz(r, c / 8, NR) + (c % 8) * 2, u32(h));
                if (v) *reinterpret_cast<__half2*>(a.H + (size_t)m * a.ldh + c) = h;
            }
        }
        __syncthreads();

        if (a.xout) {               // x_{l+1} = h . Wres^T + Bres + x_l
            float ar[NJ][4];
#pragma unroll
            for (int j = 0; j < NJ; j++)
#pragma unroll
                for (int i = 0; i < 4; i++) ar[j][i] = 0.f;
#pragma unroll
            for (int kk = 0; kk < R / 16; kk++) {
                uint32_t af[4];
                load_a(af, sHT, NR, wm * 16, 2 * kk, lane);
#pragma unroll
                for (int jj = 0; jj < NJ / 2; jj++) {
                    uint32_t b[4];
                    load_b2(b, sWr, NR, wn * (R / 2) + 16 * jj, 2 * kk, lane);
                    mma(ar[2 * jj], af, b[0], b[1]);
                    mma(ar[2 * jj + 1], af, b[2], b[3]);
                }
            }
#pragma unroll
            for (int hr = 0; hr < 2; hr++) {
                const int m = MODELS ? srow[wm * 16 + g + 8 * hr] : m0 + wm * 16 + g + 8 * hr;
                if (MODELS ? m < 0 : m >= a.M) continue;
#pragma unroll
                for (int j = 0; j < NJ; j++) {
                    const int c = wn * (R / 2) + 8 * j + 2 * q;
                    const float2 br = *reinterpret_cast<const float2*>(MODELS ? Br + c : a.Br + c);
                    float2* xp = reinterpret_cast<float2*>(a.xf + (size_t)m * R + c);
                    const float2 x = *xp;
                    const float2 y = make_float2((ar[j][2 * hr] + br.x) + x.x, (ar[j][2 * hr + 1] + br.y) + x.y);
                    *xp = y;
                    *reinterpret_cast<__half2*>(a.xout + (size_t)m * R + c) = __floats2half2_rn(y.x, y.y);
                }
            }
        }
    }
}

// ---- output: skip sum, Zs, Za, log-softmax ----
struct OutArgs {
    const __half* H;                // [M][K1]
    int K1;                         // L * R
    const __half *Ws, *Wzs, *Wza;   // [S][K1], [A][S], [A][A]
    const float *Bsk, *Bzs, *Bza;
    const int* audio;               // [Bs][N]
    int N, t0, M, Bs;
    float* logp;                    // [Bs][N]
    float* logits;                  // row (t, b) at logits + b * logits_ld + (t - logits_t0) * A, or NULL
    long long logits_ld;
    int logits_t0;
};

constexpr int STAGE = BM * KS * 2 + A_OUT * KS * 2;      // A slice + B slice of one k-step
constexpr int LG_LD = A_OUT + 8;                         // padded fp32 logit rows
constexpr int OUT_SMEM = 2 * STAGE + BM * A_OUT * 2 * 2 + BM * LG_LD * 4;

// acc (16 rows x NT * 8 columns of this warp) = A[rows][0..K) . B[N][0..K)^T with B (and A when A_GLOBAL) streamed through a
// two-stage cp.async ring in k-slices of 64; otherwise A is a resident row-major tile of a_nch chunks per row.  A's rows are
// m0 + r below M, or with MAPPED rows[r] where that is not negative
template <int NT, bool A_GLOBAL, bool MAPPED = false>
__device__ __forceinline__ void gemm_stream(float (&acc)[NT][4], const __half* __restrict__ Ag, int lda, int m0, int M, const int* rows, uint32_t sAres, int a_nch,
                                            const __half* __restrict__ Bg, int K, uint32_t ring, int tid, int lane, int wm, int wn)
{
    constexpr int N = NT * 16;
#pragma unroll
    for (int j = 0; j < NT; j++)
#pragma unroll
        for (int i = 0; i < 4; i++) acc[j][i] = 0.f;
    const int ns = (K + KS - 1) / KS;
    auto load = [&](int s) {
        const uint32_t sa = ring + (s & 1) * STAGE, sb = sa + BM * KS * 2;
        if (A_GLOBAL) {
            for (int i = tid; i < BM * 8; i += NTHREADS) {
                const int r = i / 8, c = i % 8, m = MAPPED ? rows[r] : m0 + r, k = s * KS + c * 8;
                const bool v = (MAPPED ? m >= 0 : m < M) && k < K;
                cp16(sa + swz(r, c, 8), Ag + (v ? (size_t)m * lda + k : 0), v);
            }
        }
        for (int i = tid; i < N * 8; i += NTHREADS) {
            const int n = i / 8, c = i % 8, k = s * KS + c * 8;
            const bool v = k < K;
            cp16(sb + swz(n, c, 8), Bg + (v ? (size_t)n * K + k : 0), v);
        }
        cp_commit();
    };
    load(0);
    for (int s = 0; s < ns; s++) {
        if (s + 1 < ns) { load(s + 1); cp_wait<1>(); } else cp_wait<0>();
        __syncthreads();
        const uint32_t sa = ring + (s & 1) * STAGE, sb = sa + BM * KS * 2;
#pragma unroll
        for (int kk = 0; kk < KS / 16; kk++) {
            uint32_t af[4];
            if (A_GLOBAL) load_a(af, sa, 8, wm * 16, 2 * kk, lane);
            else load_a(af, sAres, a_nch, wm * 16, s * 8 + 2 * kk, lane);
#pragma unroll
            for (int jj = 0; jj < NT / 2; jj++) {
                uint32_t b[4];
                load_b2(b, sb, 8, wn * (N / 2) + 16 * jj, 2 * kk, lane);
                mma(acc[2 * jj], af, b[0], b[1]);
                mma(acc[2 * jj + 1], af, b[2], b[3]);
            }
        }
        __syncthreads();
    }
}

// relu(acc + bias) -> fp16 row-major tile of nch chunks per row
template <int NT>
__device__ __forceinline__ void relu_to_tile(const float (&acc)[NT][4], const float* __restrict__ bias, uint32_t tile, int nch, int wm, int wn, int lane)
{
    const int g = lane >> 2, q = lane & 3;
#pragma unroll
    for (int hr = 0; hr < 2; hr++) {
        const int r = wm * 16 + g + 8 * hr;
#pragma unroll
        for (int j = 0; j < NT; j++) {
            const int c = wn * (NT * 8) + 8 * j + 2 * q;
            const float v0 = fmaxf(acc[j][2 * hr] + bias[c], 0.f), v1 = fmaxf(acc[j][2 * hr + 1] + bias[c + 1], 0.f);
            sts32(tile + swz(r, c / 8, nch) + (c % 8) * 2, u32(__floats2half2_rn(v0, v1)));
        }
    }
}

// MODELS: each tile reads its model's weights, and its rows through srow as the layer kernel's
template <int S, bool MODELS>
__global__ void __launch_bounds__(NTHREADS) score_out_kernel(const OutArgs a, const ModelArgs x)
{
    extern __shared__ __align__(128) unsigned char smem[];
    constexpr int A = A_OUT;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp & 3, wn = warp >> 2;
    const uint32_t ring = smem_u32(smem), sZ1 = ring + 2 * STAGE, sZ2 = sZ1 + BM * A * 2;
    float* lg = reinterpret_cast<float*>(smem + 2 * STAGE + 2 * BM * A * 2);
    int* srow = reinterpret_cast<int*>(smem + OUT_SMEM);

    const int tiles = MODELS ? x.tiles : (a.M + BM - 1) / BM;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int m0 = tile * BM;
        const char* im = nullptr;                     // MODELS: the tile's model's image
        if (MODELS) {
            const int T = a.M / a.Bs;
            int start;
            const int k = score_seg(x.segs, T, tile, start);
            im = static_cast<const char*>(x.segs->image[x.segs->model[k]]);
            if (tid < BM) srow[tid] = score_row(x.segs, k, (tile - start) * BM + tid, T, a.Bs);
            __syncthreads();                            // the last tile ended with a barrier: its reads of srow are done
        }
        {
            float acc[S / 16][4];
            gemm_stream<S / 16, true, MODELS>(acc, a.H, a.K1, m0, a.M, srow, 0, 0, MODELS ? reinterpret_cast<const __half*>(im + x.oWs) : a.Ws, a.K1, ring, tid, lane, wm, wn);
            relu_to_tile<S / 16>(acc, MODELS ? reinterpret_cast<const float*>(im + x.oBsk) : a.Bsk, sZ1, S / 8, wm, wn, lane);
        }
        __syncthreads();
        {
            float acc[A / 16][4];
            gemm_stream<A / 16, false>(acc, nullptr, 0, m0, a.M, nullptr, sZ1, S / 8, MODELS ? reinterpret_cast<const __half*>(im + x.oWzs) : a.Wzs, S, ring, tid, lane, wm, wn);
            relu_to_tile<A / 16>(acc, MODELS ? reinterpret_cast<const float*>(im + x.oBzs) : a.Bzs, sZ2, A / 8, wm, wn, lane);
        }
        __syncthreads();
        {
            float acc[A / 16][4];
            gemm_stream<A / 16, false>(acc, nullptr, 0, m0, a.M, nullptr, sZ2, A / 8, MODELS ? reinterpret_cast<const __half*>(im + x.oWza) : a.Wza, A, ring, tid, lane, wm, wn);
            const int g = lane >> 2, q = lane & 3;
            const float* Bza = MODELS ? reinterpret_cast<const float*>(im + x.oBza) : a.Bza;
#pragma unroll
            for (int hr = 0; hr < 2; hr++) {
                const int r = wm * 16 + g + 8 * hr;
#pragma unroll
                for (int j = 0; j < A / 16; j++) {
                    const int c = wn * (A / 2) + 8 * j + 2 * q;
                    *reinterpret_cast<float2*>(lg + r * LG_LD + c) = make_float2(acc[j][2 * hr] + Bza[c], acc[j][2 * hr + 1] + Bza[c + 1]);
                }
            }
        }
        __syncthreads();
        // log-softmax in fp32 with accurate expf / logf, one warp per row, fixed reduction trees
        for (int r = warp; r < BM; r += NTHREADS / 32) {
            const int m = MODELS ? srow[r] : m0 + r;
            if (MODELS ? m < 0 : m >= a.M) break;
            const int b = m % a.Bs, t = a.t0 + m / a.Bs;
            float z[A / 32], mx = -INFINITY;
#pragma unroll
            for (int i = 0; i < A / 32; i++) { z[i] = lg[r * LG_LD + lane + 32 * i]; mx = fmaxf(mx, z[i]); }
#pragma unroll
            for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            float s = 0.f;
#pragma unroll
            for (int i = 0; i < A / 32; i++) s += expf(z[i] - mx);
#pragma unroll
            for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            const float lse = mx + logf(s);
            if (lane == 0) {
                const size_t bt = (size_t)b * a.N + t;
                a.logp[bt] = lg[r * LG_LD + a.audio[bt]] - lse;
            }
            if (a.logits) {
                float* dst = a.logits + (size_t)b * a.logits_ld + (size_t)(t - a.logits_t0) * A;
#pragma unroll
                for (int i = 0; i < A / 32; i++) dst[lane + 32 * i] = z[i];
            }
        }
        __syncthreads();
    }
}

int num_sms()
{
    static int n = 0;
    if (!n) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n < 1) n = 1;
    }
    return n;
}

// one wave of CTAs, each looping over row tiles (the weights a CTA stages are loaded once per launch)
template <typename Args>
cudaError_t launch_persistent(void (*kernel)(Args, ModelArgs), int smem, int tiles, cudaStream_t st, const Args& args, const ModelArgs& x)
{
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    int per_sm = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, NTHREADS, smem);
    if (e != cudaSuccess) return e;
    if (per_sm < 1) return cudaErrorInvalidConfiguration;
    int grid = num_sms() * per_sm;
    if (grid > tiles) grid = tiles;
    kernel<<<grid, NTHREADS, smem, st>>>(args, x);
    return cudaGetLastError();
}

template <int R>
cudaError_t launch_layer(const LayerArgs& a, const ModelArgs& x, cudaStream_t st)
{
    static_assert(layer_smem<R>() + BM * 4 <= 227 * 1024, "layer kernel shared memory");
    if (x.segs)
        return launch_persistent(a.tau ? score_layer_kernel<R, true, true> : score_layer_kernel<R, false, true>, layer_smem<R>() + BM * 4, x.tiles, st, a, x);
    return launch_persistent(a.tau ? score_layer_kernel<R, true, false> : score_layer_kernel<R, false, false>, layer_smem<R>(), (a.M + BM - 1) / BM, st, a, x);
}

template <int S>
cudaError_t launch_out(const OutArgs& a, const ModelArgs& x, cudaStream_t st)
{
    static_assert(OUT_SMEM + BM * 4 <= 227 * 1024, "output kernel shared memory");
    if (x.segs) return launch_persistent(score_out_kernel<S, true>, OUT_SMEM + BM * 4, x.tiles, st, a, x);
    return launch_persistent(score_out_kernel<S, false>, OUT_SMEM, (a.M + BM - 1) / BM, st, a, x);
}

}  // namespace

// the oracle's dilation schedule (nv_wavenet_reference.cpp:283-293): 1, 2, 4, ... doubling per layer, back to 1 past maxDil
int wn_score_dilation(int layer, int maxDil)
{
    int d = 1;
    for (int l = 0; l < layer; l++) {
        d *= 2;
        if (d > maxDil) d = 1;
    }
    return d;
}

size_t wn_score_xh_offset(int layer, int L, int maxDil, int Tcap, int Be, int R)
{
    (void)L;
    size_t off = 0;
    for (int l = 0; l < layer; l++) off += (size_t)(wn_score_dilation(l, maxDil) + Tcap) * Be * R;
    return off;
}

size_t wn_score_image_bytes(int R, int S, int A, int L) { return image_layout(R, S, A, L).bytes; }

cudaError_t wn_score_pack(void* image, const WnParams& p, cudaStream_t st)
{
    const int R = p.R, S = p.S, A = p.A, L = p.L;
    const ImageLayout o = image_layout(R, S, A, L);
    char* im = static_cast<char*>(image);
    auto h = [](const void* q) { return static_cast<const __half*>(q); };
    const int blocks = 132 * 4;
    pack_w1_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<__half*>(im + o.W1), h(p.Wcur), h(p.Wprev), R, L);
    pack_t_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<__half*>(im + o.Wr), (size_t)R * R, R, h(p.Wres), (size_t)R * R, R, R, L);
    pack_t_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<__half*>(im + o.Ws), (size_t)R, L * R, h(p.Wskip), (size_t)S * R, S, R, L);
    pack_t_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<__half*>(im + o.Wzs), 0, S, h(p.Wzs), 0, A, S, 1);
    pack_t_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<__half*>(im + o.Wza), 0, A, h(p.Wza), 0, A, A, 1);
    pack_bias_kernel<<<4, 256, 0, st>>>(reinterpret_cast<float*>(im + o.Bh), reinterpret_cast<float*>(im + o.Br), reinterpret_cast<float*>(im + o.Bsk),
                                        reinterpret_cast<float*>(im + o.Bzs), reinterpret_cast<float*>(im + o.Bza), h(p.Bh), h(p.Bres), h(p.Bskip),
                                        h(p.Bzs), h(p.Bza), R, S, A, L);
    return cudaGetLastError();
}

cudaError_t wn_score_check_audio(const int* audio, size_t n, int A, unsigned long long* first_bad, cudaStream_t st)
{
    size_t blocks = (n + 255) / 256;
    if (blocks > 132 * 8) blocks = 132 * 8;
    if (blocks < 1) blocks = 1;
    check_audio_kernel<<<(unsigned)blocks, 256, 0, st>>>(audio, n, A, first_bad);
    return cudaGetLastError();
}

cudaError_t wn_score_carry_codes(int* codes, const int* audio, int N, int count, int Bs, cudaStream_t st)
{
    carry_codes_kernel<<<(Bs + 255) / 256, 256, 0, st>>>(codes, audio, N, count, Bs);
    return cudaGetLastError();
}

cudaError_t wn_score_chunk(const WnScoreChunk& c, cudaStream_t st)
{
    if (c.A != A_OUT || (c.S != 128 && c.S != 256) || (c.R != 32 && c.R != 64 && c.R != 128)) return cudaErrorInvalidValue;
    const ImageLayout o = image_layout(c.R, c.S, c.A, c.L);
    const char* im = static_cast<const char*>(c.image);
    const int M = c.T * c.Bs, R = c.R;
    cudaError_t e;
    if (c.starts) {
        score_tau_kernel<<<(c.Bs + 3) / 4, 128, 0, st>>>(c.tau, c.tau_carry, c.starts, c.N, c.t0, c.T, c.Bs, c.maxDil > 2 ? c.maxDil : 2);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    const int* tau = c.starts ? c.tau : nullptr;
    ModelArgs x = {};
    if (c.segs) {                                     // scoring by model: the chunk's tiles, segment by segment
        x.segs = c.segs_dev;
        for (int k = 0; k < c.segs->count; k++) x.tiles += (c.T * c.segs->n[k] + BM - 1) / BM;
        x.oWs = o.Ws; x.oWzs = o.Wzs; x.oWza = o.Wza; x.oBsk = o.Bsk; x.oBzs = o.Bzs; x.oBza = o.Bza;
    }
    {
        const size_t n = (size_t)M * R;
        size_t blocks = (n + 255) / 256;
        if (blocks > 132 * 16) blocks = 132 * 16;
        __half* x0 = c.xh + (size_t)wn_score_dilation(0, c.maxDil) * c.Bs * R;
        auto embed = c.segs ? (tau ? score_embed_kernel<true, true> : score_embed_kernel<false, true>)
                            : (tau ? score_embed_kernel<true, false> : score_embed_kernel<false, false>);
        embed<<<(unsigned)blocks, 256, 0, st>>>(static_cast<const __half*>(c.embPrev), static_cast<const __half*>(c.embCur), c.audio, c.codes, c.N, c.t0,
                                                M, c.Bs, R, c.tanhEmbed, c.xf, x0, tau, c.segs_dev);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    for (int l = 0; l < c.L; l++) {
        LayerArgs a;
        a.W1 = reinterpret_cast<const __half*>(im + o.W1) + (size_t)l * 4 * R * R;
        a.Wr = reinterpret_cast<const __half*>(im + o.Wr) + (size_t)l * R * R;
        a.Bh = reinterpret_cast<const float*>(im + o.Bh) + (size_t)l * 2 * R;
        a.Br = reinterpret_cast<const float*>(im + o.Br) + (size_t)l * R;
        a.d = wn_score_dilation(l, c.maxDil);
        a.hist = a.d * c.Bs;
        a.tau = tau;
        a.xin = c.xh + wn_score_xh_offset(l, c.L, c.maxDil, c.Tcap, c.Be, R);
        a.xf = c.xf;
        a.xout = l + 1 < c.L ? c.xh + wn_score_xh_offset(l + 1, c.L, c.maxDil, c.Tcap, c.Be, R) + (size_t)wn_score_dilation(l + 1, c.maxDil) * c.Bs * R
                             : nullptr;
        a.H = c.H + (size_t)l * R;
        a.ldh = c.L * R;
        a.lh = c.lh + (size_t)l * c.Be * 2 * R;
        a.lh_t = (size_t)c.L * c.Be * 2 * R;
        a.M = M; a.Bs = c.Bs;
        x.oW1 = o.W1 + (size_t)l * 4 * R * R * 2; x.oWr = o.Wr + (size_t)l * R * R * 2;
        x.oBh = o.Bh + (size_t)l * 2 * R * 4; x.oBr = o.Br + (size_t)l * R * 4;
        e = R == 32 ? launch_layer<32>(a, x, st) : R == 64 ? launch_layer<64>(a, x, st) : launch_layer<128>(a, x, st);
        if (e != cudaSuccess) return e;
    }
    OutArgs a;
    a.H = c.H; a.K1 = c.L * R;
    a.Ws = reinterpret_cast<const __half*>(im + o.Ws); a.Wzs = reinterpret_cast<const __half*>(im + o.Wzs); a.Wza = reinterpret_cast<const __half*>(im + o.Wza);
    a.Bsk = reinterpret_cast<const float*>(im + o.Bsk); a.Bzs = reinterpret_cast<const float*>(im + o.Bzs); a.Bza = reinterpret_cast<const float*>(im + o.Bza);
    a.audio = c.audio; a.N = c.N; a.t0 = c.t0; a.M = M; a.Bs = c.Bs;
    a.logp = c.logp; a.logits = c.logits; a.logits_ld = c.logits_ld; a.logits_t0 = c.logits_t0;
    return c.S == 128 ? launch_out<128>(a, x, st) : launch_out<256>(a, x, st);
}
