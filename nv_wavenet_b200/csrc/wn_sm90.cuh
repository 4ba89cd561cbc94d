// wn_sm90.cuh -- thin inline-PTX layer over the Hopper (sm_90a) features the tensor-core kernels use:
// mbarrier, 1-D bulk TMA (cp.async.bulk), proxy fences and warpgroup MMA (wgmma) with shared-memory operands.
// Hand-written; no CUTLASS/CuTe dependency.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace sm90 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// ------------------------------------------------------------------ mbarrier, by shared-memory address (uint64_t* forms below)
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar)
{
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
// a look that never suspends the thread (try_wait parks it until a time limit when the phase is still running)
__device__ __forceinline__ bool mbar_test_wait(uint32_t bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
// three looks issued back to back: their ~90-cycle latencies overlap
__device__ __forceinline__ void mbar_try_wait3(uint32_t b1, uint32_t p1, uint32_t b2, uint32_t p2, uint32_t b3, uint32_t p3, bool& o1, bool& o2, bool& o3)
{
    uint32_t r1, r2, r3;
    asm volatile("{\n\t.reg .pred q1, q2, q3;\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 q1, [%3], %4;\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 q2, [%5], %6;\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 q3, [%7], %8;\n\t"
                 "selp.u32 %0, 1, 0, q1;\n\tselp.u32 %1, 1, 0, q2;\n\tselp.u32 %2, 1, 0, q3;\n\t}"
                 : "=r"(r1), "=r"(r2), "=r"(r3) : "r"(b1), "r"(p1), "r"(b2), "r"(p2), "r"(b3), "r"(p3) : "memory");
    o1 = r1 != 0; o2 = r2 != 0; o3 = r3 != 0;
}
// Bounded spin: a protocol slip must surface as a launch failure with a message, never as a hung GPU.
static __device__ __noinline__ void mbar_timeout(uint32_t bar, uint32_t parity)
{
    printf("nv_wavenet: mbarrier wait timed out: block %d thread %d barrier@0x%x parity %u\n", blockIdx.x, threadIdx.x, bar, parity);
    __trap();
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity))
        if (++spins > (1u << 24)) mbar_timeout(bar, parity);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) { mbar_init(smem_u32(bar), count); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) { mbar_arrive(smem_u32(bar)); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) { mbar_arrive_expect_tx(smem_u32(bar), bytes); }
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) { return mbar_try_wait(smem_u32(bar), parity); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) { mbar_wait(smem_u32(bar), parity); }

// ------------------------------------------------------------------ fences
// generic-proxy writes (st.shared / st.global) -> visible to the async proxy (TMA, wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

// ------------------------------------------------------------------ 1-D bulk TMA: global -> shared, completes on an mbarrier
__device__ __forceinline__ void tma_load_1d(uint32_t smem_dst, const void* gmem_src, uint32_t bytes, uint32_t bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_dst), "l"(gmem_src), "r"(bytes), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar)
{
    tma_load_1d(smem_u32(smem_dst), gmem_src, bytes, smem_u32(bar));
}
// pull a global range towards L2 ahead of the TMA that will read it
__device__ __forceinline__ void tma_prefetch_l2(const void* gmem_src, uint32_t bytes)
{
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gmem_src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ uint4 ldg_nc_v4(const void* p)
{
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

// ------------------------------------------------------------------ operand tiles
// byte offset of element (row, k) inside a K-major SWIZZLE_128B tile of 64 fp16 per row (rows 128 B apart, the 16-byte
// chunks of a row XOR-permuted with row & 7); tiles are 1024-byte aligned
__host__ __device__ constexpr uint32_t sw128_offset(uint32_t row, uint32_t k)
{
    return row * 128u + ((((k >> 3) ^ (row & 7u)) << 4) | ((k & 7u) << 1));
}
// wgmma shared-memory matrix descriptor of such a tile: start address, leading byte offset 16 (unused with one swizzle atom
// along K), stride byte offset 1024 between 8-row groups, layout SWIZZLE_128B.  The K slice k (16 fp16 = 32 bytes) of a tile
// is addressed by adding 2 * k to the descriptor; rows [8 g, ...) by adding 64 * g (1024 bytes).
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t smem_addr)
{
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

// ------------------------------------------------------------------ wgmma (one warpgroup = 128 threads, all converged)
// Accumulator fragment of m64nN (N/2 floats per thread): thread i of the warpgroup holds d[4j + e] at
//   row 16 (i / 32) + (i % 32) / 4 + 8 (e / 2),  column 8 j + 2 (i % 4) + (e % 2)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// operand lists of the wgmma wrappers: "%0, %1, ..." and the matching "+f"(d[i]) constraints, eight at a time
#define WG_R8(a, b, c, e, f, g, h, k) "%" #a ", %" #b ", %" #c ", %" #e ", %" #f ", %" #g ", %" #h ", %" #k
#define WG_C8(a, b, c, e, f, g, h, k) "+f"(d[a]), "+f"(d[b]), "+f"(d[c]), "+f"(d[e]), "+f"(d[f]), "+f"(d[g]), "+f"(d[h]), "+f"(d[k])
#define WG_REGS_16 WG_R8(0, 1, 2, 3, 4, 5, 6, 7) ", " WG_R8(8, 9, 10, 11, 12, 13, 14, 15)
#define WG_CONS_16 WG_C8(0, 1, 2, 3, 4, 5, 6, 7), WG_C8(8, 9, 10, 11, 12, 13, 14, 15)
#define WG_REGS_32 WG_REGS_16 ", " WG_R8(16, 17, 18, 19, 20, 21, 22, 23) ", " WG_R8(24, 25, 26, 27, 28, 29, 30, 31)
#define WG_CONS_32 WG_CONS_16, WG_C8(16, 17, 18, 19, 20, 21, 22, 23), WG_C8(24, 25, 26, 27, 28, 29, 30, 31)
#define WG_REGS_64 WG_REGS_32 ", " WG_R8(32, 33, 34, 35, 36, 37, 38, 39) ", " WG_R8(40, 41, 42, 43, 44, 45, 46, 47) ", " WG_R8(48, 49, 50, 51, 52, 53, 54, 55) ", " WG_R8(56, 57, 58, 59, 60, 61, 62, 63)
#define WG_CONS_64 WG_CONS_32, WG_C8(32, 33, 34, 35, 36, 37, 38, 39), WG_C8(40, 41, 42, 43, 44, 45, 46, 47), WG_C8(48, 49, 50, 51, 52, 53, 54, 55), WG_C8(56, 57, 58, 59, 60, 61, 62, 63)
#define WG_REGS_128 WG_REGS_64 ", " WG_R8(64, 65, 66, 67, 68, 69, 70, 71) ", " WG_R8(72, 73, 74, 75, 76, 77, 78, 79) ", " WG_R8(80, 81, 82, 83, 84, 85, 86, 87) ", " WG_R8(88, 89, 90, 91, 92, 93, 94, 95) ", " WG_R8(96, 97, 98, 99, 100, 101, 102, 103) ", " WG_R8(104, 105, 106, 107, 108, 109, 110, 111) ", " WG_R8(112, 113, 114, 115, 116, 117, 118, 119) ", " WG_R8(120, 121, 122, 123, 124, 125, 126, 127)
#define WG_CONS_128 WG_CONS_64, WG_C8(64, 65, 66, 67, 68, 69, 70, 71), WG_C8(72, 73, 74, 75, 76, 77, 78, 79), WG_C8(80, 81, 82, 83, 84, 85, 86, 87), WG_C8(88, 89, 90, 91, 92, 93, 94, 95), WG_C8(96, 97, 98, 99, 100, 101, 102, 103), WG_C8(104, 105, 106, 107, 108, 109, 110, 111), WG_C8(112, 113, 114, 115, 116, 117, 118, 119), WG_C8(120, 121, 122, 123, 124, 125, 126, 127)
// D[64 x N] (fp32, registers) (+)= A[64 x 16] . B[N x 16]^T, both operands K-major SWIZZLE_128B in shared memory
#define WG_MMA(N, R, OA, OB, OP, REGS, CONS)                                                                                      \
    __device__ __forceinline__ void wgmma_m64n##N(float (&d)[R], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) \
    {                                                                                                                   \
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #OP ", 0;\n\t"                                     \
                     "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.f16.f16 {" REGS "}, %" #OA ", %" #OB ", p, 1, 1, 0, 0;\n\t}" \
                     : CONS                                                                                             \
                     : "l"(desc_a), "l"(desc_b), "r"(accumulate));                                                      \
    }
WG_MMA(32, 16, 16, 17, 18, WG_REGS_16, WG_CONS_16)
WG_MMA(64, 32, 32, 33, 34, WG_REGS_32, WG_CONS_32)
WG_MMA(128, 64, 64, 65, 66, WG_REGS_64, WG_CONS_64)
WG_MMA(256, 128, 128, 129, 130, WG_REGS_128, WG_CONS_128)
#undef WG_MMA

template <int N>
__device__ __forceinline__ void wgmma_f16(float (&d)[N / 2], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate)
{
    static_assert(N == 32 || N == 64 || N == 128 || N == 256, "wgmma_f16: N");
    if constexpr (N == 32) wgmma_m64n32(d, desc_a, desc_b, accumulate);
    else if constexpr (N == 64) wgmma_m64n64(d, desc_a, desc_b, accumulate);
    else if constexpr (N == 128) wgmma_m64n128(d, desc_a, desc_b, accumulate);
    else wgmma_m64n256(d, desc_a, desc_b, accumulate);
}

}  // namespace sm90
