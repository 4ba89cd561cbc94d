// wn_layout.cuh -- the layout operations of WnFamily (wn_common.h), written once for every kernel family's layouts.
//
// A layout is a struct next to its family's kernel.  It says where the channels of one utterance row sit, in units: the channels one
// thread moves in one memory access.
//   TD                                    element type of the conditioning store and the history ring
//   STORE_UNIT, RING_UNIT                 channels per unit; a unit is a WnVec<TD, UNIT>
//   store_unit(c, store, sl, b, k)        unit k of row b of the store at sl = position * L + layer, at the engine's batch c.B
//   ring_unit(c, ring, e, stride, b, k)   unit k of row b of ring entry e = slot * L + layer; stride is the batch stride of the plain
//                                         ring (the engine's B for clear_rows and the per-slot writers, the run's batch for the
//                                         whole-batch history writers), which the tiled layouts ignore
//   store_bytes(c), ring_bytes(c)
// Every operation below finds its units through these two functions and nothing else.  So convert_rows writes what convert writes,
// bit for bit, and a row operation touches the units of its rows and no other byte.
#pragma once
#include "wn_common.h"

// N elements of T, aligned so that one unit is one load or store (up to 16 bytes)
template <typename T, int N>
struct alignas(N * sizeof(T) < 16 ? N * sizeof(T) : 16) WnVec {
    T v[N];
};

// A unit loaded in whole words of up to 16 bytes: nvcc copies a struct of fp16 or fp32 elements element by element.
template <int BYTES> struct WnWord;
template <> struct WnWord<2> { using type = unsigned short; };
template <> struct WnWord<4> { using type = unsigned; };
template <> struct WnWord<8> { using type = uint2; };
template <> struct WnWord<16> { using type = uint4; };
template <typename T, int N>
__device__ __forceinline__ WnVec<T, N> wn_load(const WnVec<T, N>* p)
{
    constexpr int BYTES = N * sizeof(T), W = BYTES < 16 ? BYTES : 16;
    using Word = typename WnWord<W>::type;
    WnVec<T, N> u;
#pragma unroll
    for (int k = 0; k < BYTES / W; k++) reinterpret_cast<Word*>(&u)[k] = reinterpret_cast<const Word*>(p)[k];
    return u;
}

__device__ __forceinline__ void wn_cvt(float& d, float s) { d = s; }
__device__ __forceinline__ void wn_cvt(__half& d, float s) { d = __float2half_rn(s); }
__device__ __forceinline__ void wn_cvt(float& d, __half s) { d = __half2float(s); }
__device__ __forceinline__ void wn_cvt(__half& d, __half s) { d = s; }

template <typename TO, typename TI, int N>
__device__ __forceinline__ WnVec<TO, N> wn_vec_cast(const WnVec<TI, N>& a)
{
    WnVec<TO, N> o;
#pragma unroll
    for (int j = 0; j < N; j++) wn_cvt(o.v[j], a.v[j]);
    return o;
}

// One grid rule for every layout kernel: blocks of 256 threads, at most four waves of full occupancy on the H100's 132 SMs; the
// kernels' loops stride over the rest.
template <typename... P, typename... Args>
cudaError_t wn_layout_launch(void (*kernel)(size_t, P...), size_t total, cudaStream_t stream, Args... args)
{
    if (total == 0) return cudaSuccess;
    const size_t blocks = (total + 255) / 256;
    kernel<<<(unsigned)(blocks < 132 * 32 ? blocks : 132 * 32), 256, 0, stream>>>(total, args...);
    return cudaGetLastError();
}

// Thread i moves unit i % units of row i / units.  units, the units of R or 2R channels, is a power of two (R is 32, 64 or 128:
// wn_stream_supported, wn_tc_supported, wn_lat_supported), so the split is a shift and a mask: a division per element would make
// these kernels instruction-bound.
__device__ __forceinline__ int wn_log2(int units) { return __ffs(units) - 1; }

// fp32 [num_pos][L][n][2R] -> rows rows[r] (rows NULL: row r) of store positions [first_pos, first_pos + num_pos)
template <class Lay>
__global__ void wn_convert_rows_kernel(size_t total, WnConfig c, void* store, const float* __restrict__ src, const int* __restrict__ rows, int n,
                                       int first_pos)
{
    constexpr int U = Lay::STORE_UNIT;
    const int units = 2 * c.R / U, lg = wn_log2(units);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t row = i >> lg;                                   // (s * L + l) * n + r
        const int r = (int)(row % n);
        *Lay::store_unit(c, store, (size_t)first_pos * c.L + row / n, rows ? rows[r] : r, (int)i & (units - 1)) =
            wn_vec_cast<typename Lay::TD>(wn_load(reinterpret_cast<const WnVec<float, U>*>(src) + i));
    }
}

// store positions [first_pos, first_pos + num_pos) -> fp32 [num_pos][L][B][2R]
template <class Lay>
__global__ void wn_readback_kernel(size_t total, WnConfig c, float* __restrict__ dst, const void* store, int first_pos)
{
    constexpr int U = Lay::STORE_UNIT;
    const int units = 2 * c.R / U, lg = wn_log2(units);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t row = i >> lg;                                   // (s * L + l) * B + b
        reinterpret_cast<WnVec<float, U>*>(dst)[i] =
            wn_vec_cast<float>(wn_load(Lay::store_unit(c, const_cast<void*>(store), (size_t)first_pos * c.L + row / c.B, (int)(row % c.B), (int)i & (units - 1))));
    }
}

// rows rows[r] zeroed in every ring entry, at the engine's batch stride
template <class Lay>
__global__ void wn_clear_rows_kernel(size_t total, WnConfig c, void* ring, const int* __restrict__ rows, int n)
{
    const int units = c.R / Lay::RING_UNIT, lg = wn_log2(units);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t row = i >> lg;                                   // e * n + r
        *Lay::ring_unit(c, ring, row / n, c.B, rows[row % n], (int)i & (units - 1)) = WnVec<typename Lay::TD, Lay::RING_UNIT>{};
    }
}

// fp16 src [n][batch][R] -> rows 0..batch-1 of entries (t mod (maxDil+1)) * L + layer, t = t_first + j, at the batch stride `batch`
template <class Lay>
__global__ void wn_put_history_kernel(size_t total, WnConfig c, void* ring, const __half* __restrict__ src, int layer, long long t_first, int batch)
{
    constexpr int U = Lay::RING_UNIT;
    const int units = c.R / U, lg = wn_log2(units);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t row = i >> lg;                                   // j * batch + b
        const long long t = t_first + (long long)(row / batch);
        *Lay::ring_unit(c, ring, (size_t)(t % (c.maxDil + 1)) * c.L + layer, batch, (int)(row % batch), (int)i & (units - 1)) =
            wn_vec_cast<typename Lay::TD>(wn_load(reinterpret_cast<const WnVec<__half, U>*>(src) + i));
    }
}

// The ring slot of absolute time t, which may be negative here (a slot primed before the engine's sample 0, DESIGN.md §6):
// ((t mod M) + M) mod M, M = maxDil + 1.  wn_put_history_kernel's t % M is only right for t >= 0.
__device__ __forceinline__ int wn_ring_slot(long long t, int M) { return (int)((t % M + M) % M); }

// rows src_row(r) of src (the ring's type; src_rows NULL: row r) -> ring rows rows[r] of entries slot(t) * L + layer, t = t_first + j,
// at the engine's batch stride; time j of source row q at element q * row_pitch + j * time_pitch
template <class Lay>
__global__ void wn_put_history_rows_kernel(size_t total, WnConfig c, void* ring, const void* __restrict__ src, const int* __restrict__ src_rows,
                                           size_t row_pitch, size_t time_pitch, const int* __restrict__ rows, int n, int layer, long long t_first)
{
    constexpr int U = Lay::RING_UNIT;
    using TD = typename Lay::TD;
    const int units = c.R / U, lg = wn_log2(units);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t row = i >> lg;                                   // j * n + r
        const int r = (int)(row % n), k = (int)i & (units - 1);
        const size_t j = row / n;
        const size_t q = src_rows ? (size_t)src_rows[r] : (size_t)r;
        *Lay::ring_unit(c, ring, (size_t)wn_ring_slot(t_first + (long long)j, c.maxDil + 1) * c.L + layer, c.B, rows[r], k) =
            wn_load(reinterpret_cast<const WnVec<TD, U>*>(static_cast<const TD*>(src) + q * row_pitch + j * time_pitch) + k);
    }
}

// ring rows rows[r] of entries slot(t) * L + layer, t = t_first + j, at the engine's batch stride -> dst row r (the ring's type),
// time j at element r * row_pitch + j * time_pitch; zeros for the times before origin[rows[r]], whose ring bytes may be stale
template <class Lay>
__global__ void wn_get_history_rows_kernel(size_t total, WnConfig c, const void* ring, void* __restrict__ dst, size_t row_pitch, size_t time_pitch,
                                           const int* __restrict__ rows, int n, int layer, long long t_first, const long long* __restrict__ origin)
{
    constexpr int U = Lay::RING_UNIT;
    using V = WnVec<typename Lay::TD, U>;
    const int units = c.R / U, lg = wn_log2(units);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t row = i >> lg;                                   // j * n + r
        const int r = (int)(row % n), k = (int)i & (units - 1);
        const size_t j = row / n;
        const long long t = t_first + (long long)j;
        const int b = rows[r];
        V v{};
        if (t >= origin[b])
            v = wn_load(Lay::ring_unit(c, const_cast<void*>(ring), (size_t)wn_ring_slot(t, c.maxDil + 1) * c.L + layer, c.B, b, k));
        reinterpret_cast<V*>(static_cast<typename Lay::TD*>(dst) + r * row_pitch + j * time_pitch)[k] = v;
    }
}

// every row 0..B-1 of every layer's entries slot(t), t in [t_first, t_first + n_t), zeroed at the engine's batch stride
template <class Lay>
__global__ void wn_clear_times_kernel(size_t total, WnConfig c, void* ring, long long t_first)
{
    const int units = c.R / Lay::RING_UNIT, lg = wn_log2(units);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t row = i >> lg;                                   // (j * L + l) * B + b
        const size_t jl = row / c.B;
        const int l = (int)(jl % c.L);
        const long long t = t_first + (long long)(jl / c.L);
        *Lay::ring_unit(c, ring, (size_t)wn_ring_slot(t, c.maxDil + 1) * c.L + l, c.B, (int)(row % c.B), (int)i & (units - 1)) =
            WnVec<typename Lay::TD, Lay::RING_UNIT>{};
    }
}

// every ring entry -> fp32 [entries][batch][R]: rows 0..batch-1 at the batch stride `batch`, or (rows not NULL) rows rows[r] at the
// engine's batch stride
template <class Lay>
__global__ void wn_get_history_kernel(size_t total, WnConfig c, float* __restrict__ dst, const void* ring, int batch, const int* __restrict__ rows)
{
    constexpr int U = Lay::RING_UNIT;
    const int units = c.R / U, lg = wn_log2(units);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t row = i >> lg;                                   // e * batch + r
        const int r = (int)(row % batch);
        reinterpret_cast<WnVec<float, U>*>(dst)[i] = wn_vec_cast<float>(
            wn_load(Lay::ring_unit(c, const_cast<void*>(ring), row / batch, rows ? c.B : batch, rows ? rows[r] : r, (int)i & (units - 1))));
    }
}

// the WnFamily entries (wn_common.h states their contracts)
template <class Lay>
cudaError_t wn_convert_rows(const WnConfig& c, void* store, const float* src, const int* rows_dev, int n, int first_pos, int num_pos, cudaStream_t stream)
{
    return wn_layout_launch(wn_convert_rows_kernel<Lay>, (size_t)num_pos * c.L * n * (2 * c.R / Lay::STORE_UNIT), stream, c, store, src, rows_dev, n,
                            first_pos);
}
template <class Lay>
cudaError_t wn_convert(const WnConfig& c, void* store, const float* src, int first_sample, int num_samples, cudaStream_t stream)
{
    return wn_convert_rows<Lay>(c, store, src, nullptr, c.B, first_sample, num_samples, stream);
}
template <class Lay>
cudaError_t wn_readback(const WnConfig& c, float* dst_dev, const void* store, int first_sample, int num_samples, cudaStream_t stream)
{
    return wn_layout_launch(wn_readback_kernel<Lay>, (size_t)num_samples * c.L * c.B * (2 * c.R / Lay::STORE_UNIT), stream, c, dst_dev, store,
                            first_sample);
}
template <class Lay>
cudaError_t wn_clear_rows(const WnConfig& c, void* ring, const int* rows_dev, int n, cudaStream_t stream)
{
    return wn_layout_launch(wn_clear_rows_kernel<Lay>, (size_t)(c.maxDil + 1) * c.L * n * (c.R / Lay::RING_UNIT), stream, c, ring, rows_dev, n);
}
template <class Lay>
cudaError_t wn_put_history(const WnConfig& c, void* ring, const __half* src, int layer, long long t_first, int n, int batch, cudaStream_t stream)
{
    return wn_layout_launch(wn_put_history_kernel<Lay>, (size_t)n * batch * (c.R / Lay::RING_UNIT), stream, c, ring, src, layer, t_first, batch);
}
template <class Lay>
cudaError_t wn_put_history_rows(const WnConfig& c, void* ring, const void* src, const int* src_rows_dev, size_t row_pitch, size_t time_pitch,
                                const int* rows_dev, int n, int layer, long long t_first, int n_t, cudaStream_t stream)
{
    return wn_layout_launch(wn_put_history_rows_kernel<Lay>, (size_t)n_t * n * (c.R / Lay::RING_UNIT), stream, c, ring, src, src_rows_dev, row_pitch,
                            time_pitch, rows_dev, n, layer, t_first);
}
template <class Lay>
cudaError_t wn_get_history_rows(const WnConfig& c, const void* ring, void* dst, size_t row_pitch, size_t time_pitch, const int* rows_dev, int n,
                                int layer, long long t_first, int n_t, const long long* origin_dev, cudaStream_t stream)
{
    return wn_layout_launch(wn_get_history_rows_kernel<Lay>, (size_t)n_t * n * (c.R / Lay::RING_UNIT), stream, c, ring, dst, row_pitch, time_pitch,
                            rows_dev, n, layer, t_first, origin_dev);
}
template <class Lay>
cudaError_t wn_clear_times(const WnConfig& c, void* ring, long long t_first, int n_t, cudaStream_t stream)
{
    return wn_layout_launch(wn_clear_times_kernel<Lay>, (size_t)n_t * c.L * c.B * (c.R / Lay::RING_UNIT), stream, c, ring, t_first);
}
template <class Lay>
cudaError_t wn_get_history(const WnConfig& c, float* dst, const void* ring, int batch, const int* rows_dev, cudaStream_t stream)
{
    return wn_layout_launch(wn_get_history_kernel<Lay>, (size_t)(c.maxDil + 1) * c.L * batch * (c.R / Lay::RING_UNIT), stream, c, dst, ring, batch,
                            rows_dev);
}
