// wn_tc_selftest.cu -- minimal wgmma GEMM used by tests/test_gpu_tc_primitives.py to pin the operand layouts,
// descriptors and synchronisation idioms the tensor-core WaveNet kernel is built from:
//     D[128 x N] (fp32, registers) = A[128 x K] (fp16, written row-per-thread into K-major SWIZZLE_128B tiles)
//                                  x B[N x K]^T (fp16, pre-tiled image brought in by 1-D bulk TMA)
// Two warpgroups, one per 64-row half of A, as in the real kernel; thread 0 issues the TMA.
#include "wn_common.h"
#include "wn_sm90.cuh"

namespace {

using namespace sm90;

constexpr int TILE_BYTES = 128 * 128;      // [128 rows x 64 fp16] K-major SW128

// B image: for kt in K/64: for nc in N/128 (or one chunk of N rows if N < 128): tile [rows x 64]
__global__ void pack_b_kernel(const __half* __restrict__ B, int N, int K, unsigned char* __restrict__ img)
{
    const int rows_per_chunk = N < 128 ? N : 128;
    const int chunks_n = N / rows_per_chunk;
    const int total = N * K;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int n = i / K, k = i % K;
        const int kt = k / 64, kk = k % 64, nc = n / rows_per_chunk, nn = n % rows_per_chunk;
        const size_t chunk = (size_t)kt * chunks_n + nc;
        *reinterpret_cast<__half*>(img + chunk * TILE_BYTES + sw128_offset(nn, kk)) = B[i];
    }
}

// D columns [col0, col0 + NW) of this warpgroup's 64 rows = A . (NW rows of B starting at chunk c0 of every K tile)^T
template <int NW>
__device__ __forceinline__ void gemm_rows(const unsigned char* a_tiles, const unsigned char* b_tiles, int KT, int chunks_n, int c0,
                                          int wg, float* __restrict__ D, int N, int col0)
{
    float acc[NW / 2];
    wgmma_fence();
    for (int kt = 0; kt < KT; kt++) {
        const uint64_t da = make_desc_sw128(smem_u32(a_tiles + (size_t)kt * TILE_BYTES + (size_t)wg * 64 * 128));
        const uint64_t db = make_desc_sw128(smem_u32(b_tiles + (size_t)(kt * chunks_n + c0) * TILE_BYTES));
#pragma unroll
        for (int k = 0; k < 4; k++) wgmma_f16<NW>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (kt | k) ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    const int i = threadIdx.x & 127;
    const int r0 = wg * 64 + 16 * (i >> 5) + ((i & 31) >> 2), cq = 2 * (i & 3);
#pragma unroll
    for (int j = 0; j < NW / 8; j++)
#pragma unroll
        for (int e = 0; e < 4; e++) D[(size_t)(r0 + 8 * (e >> 1)) * N + col0 + 8 * j + cq + (e & 1)] = acc[4 * j + e];
}

__global__ void __launch_bounds__(256, 1) wgmma_selftest_kernel(const __half* __restrict__ A, const unsigned char* __restrict__ Bimg,
                                                                int N, int K, float* __restrict__ D, int mode)
{
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int KT = K / 64;
    const int rows_per_chunk = N < 128 ? N : 128;
    const int chunks_n = N / rows_per_chunk;
    unsigned char* a_tiles = smem;                               // KT tiles
    unsigned char* b_tiles = smem + (size_t)KT * TILE_BYTES;     // KT * chunks_n tiles
    uint64_t* b_full = reinterpret_cast<uint64_t*>(b_tiles + (size_t)KT * chunks_n * TILE_BYTES);

    const int tid = threadIdx.x, wg = tid >> 7;
    if (tid == 0) {
        mbar_init(b_full, 1);
        fence_mbar_init();
    }
    __syncthreads();
    if (tid == 0) {
        const uint32_t bytes = (uint32_t)(KT * chunks_n) * (uint32_t)(rows_per_chunk * 128);
        mbar_arrive_expect_tx(b_full, bytes);
        for (int c = 0; c < KT * chunks_n; c++)
            tma_load_1d(b_tiles + (size_t)c * TILE_BYTES, Bimg + (size_t)c * TILE_BYTES, rows_per_chunk * 128, b_full);
    }
    if (tid < 128) {
        // each thread writes its own row of A into every K tile (8 x 16-byte chunks per tile), as the kernel's epilogue does
        const int row = tid;
        for (int kt = 0; kt < KT; kt++) {
            const uint4* src = reinterpret_cast<const uint4*>(A + (size_t)row * K + kt * 64);
            for (int j = 0; j < 8; j++) {
                const uint4 v = src[j];
                *reinterpret_cast<uint4*>(a_tiles + (size_t)kt * TILE_BYTES + row * 128 + ((j ^ (row & 7)) << 4)) = v;
            }
        }
    }
    fence_proxy_async_smem();
    __syncthreads();
    mbar_wait(b_full, 0);
    if (mode == 0) {
        // one instruction per 128-row chunk of B (or the whole of a smaller B): D columns [nc * 128, ...)
        for (int nc = 0; nc < chunks_n; nc++) {
            if (rows_per_chunk == 64) gemm_rows<64>(a_tiles, b_tiles, KT, chunks_n, nc, wg, D, N, nc * 128);
            else gemm_rows<128>(a_tiles, b_tiles, KT, chunks_n, nc, wg, D, N, nc * 128);
        }
    } else {
        // N = 256 as ONE instruction per K slice: the two 128-row chunks of a K tile are contiguous (SBO walks across)
        if (N == 256) gemm_rows<256>(a_tiles, b_tiles, KT, chunks_n, 0, wg, D, N, 0);
        else gemm_rows<128>(a_tiles, b_tiles, KT, chunks_n, 0, wg, D, N, 0);
    }
}

}  // namespace

// A: [128][K] fp16 row-major, B: [N][K] fp16 row-major, D: [128][N] fp32; all HOST pointers.  K % 64 == 0,
// N in {64, 128, 256}.  mode 0: N<=128-wide instructions per 128-row chunk; mode 1: one N-wide instruction.
extern "C" int nvwn_selftest_umma(const void* A, const void* B, int N, int K, float* D, int mode)
{
    if (K % 64 || (N != 64 && N != 128 && N != 256) || K > 256 || (mode != 0 && N == 64)) return -1;
    __half *dA = nullptr, *dB = nullptr;
    unsigned char* img = nullptr;
    float* dD = nullptr;
    cudaError_t e;
#define ST(x) if ((e = (x)) != cudaSuccess) { fprintf(stderr, "selftest: %s at line %d\n", cudaGetErrorString(e), __LINE__); return (int)e; }
    ST(cudaMalloc(&dA, 128 * K * 2)); ST(cudaMalloc(&dB, (size_t)N * K * 2)); ST(cudaMalloc(&dD, 128 * N * 4));
    const int chunks = (K / 64) * (N < 128 ? 1 : N / 128);
    ST(cudaMalloc(&img, (size_t)chunks * TILE_BYTES));
    ST(cudaMemset(img, 0, (size_t)chunks * TILE_BYTES));
    ST(cudaMemcpy(dA, A, 128 * K * 2, cudaMemcpyHostToDevice));
    ST(cudaMemcpy(dB, B, (size_t)N * K * 2, cudaMemcpyHostToDevice));
    pack_b_kernel<<<64, 256>>>(dB, N, K, img);
    const size_t smem = 1024 + (size_t)(K / 64) * TILE_BYTES + (size_t)chunks * TILE_BYTES + 64;
    ST(cudaFuncSetAttribute(wgmma_selftest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    wgmma_selftest_kernel<<<1, 256, smem>>>(dA, img, N, K, dD, mode);
    ST(cudaGetLastError());
    ST(cudaDeviceSynchronize());
    ST(cudaMemcpy(D, dD, 128 * N * 4, cudaMemcpyDeviceToHost));
#undef ST
    cudaFree(dA); cudaFree(dB); cudaFree(dD); cudaFree(img);
    return 0;
}
