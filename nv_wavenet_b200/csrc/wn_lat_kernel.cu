// wn_lat_kernel.cu -- latency-mode fp16 kernel of the WaveNet inference loop (sm_90a).
//
// The autoregressive loop is a chain of ~45 tiny dependent GEMMs per sample (M = utterances, N <= 256, K <= 256).  On such a
// chain the round trip between the tensor cores and the epilogue of every link is the cost, not the tensor pipe.  This kernel
// keeps the whole chain in REGISTERS: warp-level mma.sync
// (m16n8k16, fp16 x fp16 -> fp32) with the utterances as the M dimension, so that the accumulator fragment of one GEMM is
// -- after the row-local epilogue -- exactly the A fragment of the next one; the only exchange between the eight compute
// warps is one 2 KB shared-memory tile + one named barrier per GEMM stage.
//
//   one persistent CTA per tile of 16 utterances (B = 64 -> 4 SMs), 8 compute warps + 1 producer warp:
//   compute warp w  owns output channels [8w, 8w+8) (+R for the sigmoid half) of every layer GEMM, [32w, 32w+32) of the skip
//                   sum / Zs / Za; residual stream (fp32) and skip sum (fp32) never leave its registers.
//                   per layer:  a = Wcur.x + Wprev.x[t-d] + (Bh + Lh)  ->  h = tanh * sigmoid  -> [h tile, barrier]
//                               x' = Wres.h + Bres + x -> [x tile, history ring, barrier];  skip += Wskip.h
//                   per sample: relu(skip) -> Zs -> Za -> softmax + categorical sample (warp-local, two utterances per warp)
//                               -> embedding gather from the shared-memory resident table.
//   producer warp   streams the weight image (pre-arranged in mma B-fragment order, so that every weight load of a warp is one
//                   conflict-free 512-byte LDS.128) from L2 through a shared-memory ring with bulk TMA + mbarriers: two pieces
//                   per layer ([Wcur_l | Wprev_l+1] 32 KB, [Wres_l | Wskip_l] 40 KB), two slots per piece type, every slot
//                   refilled as soon as its occupant is consumed -- each piece is in flight two layers before its use.
//   Lh (the only HBM stream), biases and the dilated history x[t-d] are prefetched into registers one / two layers ahead.
//
// wn_lat2_kernel (second half of this file, the default up to ~720 utterances) spreads the same data flow over a cluster of three
// CTAs per tile -- chain / tail / prep -- that hand tiles over through distributed shared memory; see the comment there.  The
// K = 64 gate GEMM (except the chain CTA's Wcur.x), the gate, the residual GEMM and update with the x-tile / history-ring store, the xtOut dump, the relu(skip + Bskip)
// packing and the final index store are defined once ("stages of both latency kernels") and called by both, with the trace
// points between the calls; the mbarrier / bulk-TMA wrappers come from wn_sm90.cuh.
// Each kernel body is a prologue (barriers, tables) and a dispatch to one function per role: lat_producer / lat_compute, and
// chain_cta / tail_cta / prep_cta of the cluster, which share load_out_w and out_half.  What the roles share is set once, in a
// LatCta / ClusterCta; the mbarrier maps (Cfg::B_*, CfgC::B_*) and the slot arithmetic follow from the slot counts.
//
// Replaces nv_wavenet_{singleblock,dualblock,persistent}.cuh + matrix_math.cuh + softmax.cuh of the reference for
// T_data = half while the batch is small enough to be latency-bound.  Numerical contract: oracle/wavenet_oracle.c
// WNO_PREC_FP16 (GEMM inputs fp16, fp32 accumulation, fp32 residual stream / skip sum / softmax), gate evaluated with
// tanh.approx.f16x2; no weight folding.
#include "wn_common.h"
#include "wn_layout.cuh"
#include "wn_math.cuh"
#include "wn_sm90.cuh"

#include <stdlib.h>

namespace {

using namespace sm90;

constexpr int R = 64, A = 256;
constexpr int NCW = 8;                      // compute warps
constexpr int NCT = NCW * 32;
constexpr int NT = NCT + 32;                // + producer warp
constexpr int TU = 16;                      // utterances per tile = M of mma.m16n8k16
constexpr int LROW = 264;                   // padded row (floats) of the transposed-logits buffer
constexpr int EROW = 33;                    // padded row (32-bit words) of the shared-memory embedding table
constexpr int MAXL = 64;

template <int S>
struct Cfg {
    // one layer block of the weight image = two ring pieces, in consumption order:
    //   P1 = [ Wcur_l | Wprev_{(l+1) mod L} ]  (32 KB)      P2 = [ Wres_l | Wskip_l ]  (8 KB + S x 128 B)
    static constexpr int W_CUR = 0, W_PREV = 16384, W_RES = 32768, W_SKIP = 40960;
    static constexpr int P1_BYTES = 32768, P2_BYTES = 8192 + S * 128;
    // output GEMMs: 4 + 4 ring pieces per sample, each all 32 n-tiles x OJP k-step pairs
    static constexpr int NQ_ZS = 4, NQ_ZA = 4, NQ = NQ_ZS + NQ_ZA;
    static_assert(NQ == 8, "the ring bookkeeping assumes 8 output pieces per sample");
    static constexpr int OJP_ZS = S / 128, OJP_ZA = A / 128;         // k-step pairs per piece
    static constexpr int ZS_PIECE = 32 * OJP_ZS * 512, ZA_PIECE = 32 * OJP_ZA * 512;
    static constexpr int OPIECE = ZA_PIECE > ZS_PIECE ? ZA_PIECE : ZS_PIECE;
    static constexpr int NSK = S / 64;                               // skip n-tiles per warp
    // ring: two slots per piece type; output pieces alternate between the two types
    static constexpr int SLOT1 = P1_BYTES, SLOT2 = P2_BYTES > OPIECE ? P2_BYTES : OPIECE;
    static constexpr int NSLOT = 4;                                  // ring slots of both types: piece n sits in slot (n >> 1) & 1 of type n & 1
    static constexpr int NPST = 3;                                   // staged history tiles
    // shared memory map
    static constexpr uint32_t O_RING1 = 0;                           // 2 x SLOT1
    static constexpr uint32_t O_RING2 = 2 * SLOT1;                   // 2 x SLOT2
    static constexpr uint32_t O_EMB = O_RING2 + 2 * SLOT2;
    static constexpr uint32_t O_BOUT = O_EMB + A * EROW * 4;         // fp32: Bskip total [S], Bzs [A], Bza [A]
    static constexpr uint32_t O_EPBUF = O_BOUT + (S + 2 * A) * 4;           // two [16 rows][33 words] buffers (sample parity)
    static constexpr uint32_t O_PST = O_EPBUF + 2 * TU * EROW * 4;          // NPST x 2 KB: staged history tiles x[t-d] (A-fragment order)
    static constexpr uint32_t O_OB0 = O_PST + NPST * 2048;
    static constexpr uint32_t O_OB1 = O_OB0 + (S / 16) * 512;
    static constexpr uint32_t O_LBUF = O_OB1 + (A / 16) * 512;              // transposed logits; its first 4 KB double as ...
    static constexpr uint32_t O_XBUF = O_LBUF, O_HBUF = O_LBUF + 2048;      // ... the x and h exchange tiles (dead while the logits live)
    static constexpr uint32_t O_DIL = O_LBUF + TU * LROW * 4;
    static constexpr uint32_t O_YS = O_DIL + MAXL * 4;
    static constexpr uint32_t O_BAR = O_YS + 2 * TU * 4;
    static constexpr uint32_t SMEM = O_BAR + 16 * 8;
    // mbarriers at O_BAR: ring full[NSLOT] / empty[NSLOT] (slot i of piece type k: k * 2 + i), pfull[NPST] (staged history tiles)
    static constexpr uint32_t B_FULL = 0, B_EMPTY = B_FULL + NSLOT * 8, B_PFULL = B_EMPTY + NSLOT * 8, B_END = B_PFULL + NPST * 8;
    static_assert(O_BAR + B_END <= SMEM, "the mbarriers outgrow their reservation");
    // offset of the barrier of slot i of piece type k inside full[] / empty[]
    static __device__ __forceinline__ uint32_t ring_bar(uint32_t k, uint32_t i) { return (k * 2 + i) * 8; }
};

struct LatImage {
    size_t layer_bytes, off_zs, off_za, off_bias, total;
    size_t b_layer, b_skpre, b_bzs, b_bza;      // float offsets inside the bias block
};
__host__ __device__ inline LatImage lat_image(int S, int L)
{
    LatImage im;
    im.layer_bytes = 40960 + (size_t)S * 128;
    im.off_zs = (size_t)L * im.layer_bytes;
    im.off_za = im.off_zs + (size_t)A * S * 2;
    im.off_bias = im.off_za + (size_t)A * A * 2;
    im.b_layer = 0;                             // [L][8 warps][4 t][8]: Bh tanh pair, Bh sigmoid pair, Bres pair, 0, 0
    im.b_skpre = (size_t)L * 256;               // [L][S] running sum of the skip biases
    im.b_bzs = im.b_skpre + (size_t)L * S;
    im.b_bza = im.b_bzs + A;
    im.total = im.off_bias + (im.b_bza + A) * sizeof(float);
    return im;
}

// ------------------------------------------------------------------------------------------------ device helpers
__device__ __forceinline__ void hmma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
{
    asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint4 lds128(uint32_t addr)
{
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t addr)
{
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ uint2 lds64(uint32_t addr)
{
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void sts64(uint32_t addr, uint32_t a, uint32_t b)
{
    asm volatile("st.shared.v2.u32 [%0], {%1,%2};" ::"r"(addr), "r"(a), "r"(b) : "memory");
}
__device__ __forceinline__ void sts128(uint32_t addr, uint4 v)
{
    asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void sts32(uint32_t addr, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
__device__ __forceinline__ void load_a(uint32_t (&a)[4], uint32_t addr)
{
    const uint4 v = lds128(addr);
    a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w;
}
// predicated load into an existing register quad: no select on the loaded value, so nothing waits for the load here
__device__ __forceinline__ void ldg_nc_v4_if(uint4& d, const void* p, bool pred)
{
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %5, 0;\n\t@q ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];\n\t}"
                 : "+r"(d.x), "+r"(d.y), "+r"(d.z), "+r"(d.w) : "l"(p), "r"((uint32_t)pred) : "memory");
}
__device__ __forceinline__ void stg_v2(void* p, uint32_t a, uint32_t b) { asm volatile("st.global.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(a), "r"(b) : "memory"); }
__device__ __forceinline__ void stg_b32(void* p, uint32_t a) { asm volatile("st.global.u32 [%0], %1;" ::"l"(p), "r"(a) : "memory"); }
__device__ __forceinline__ void bar_compute() { asm volatile("bar.sync 1, %0;" ::"n"(NCT) : "memory"); }
// the cluster kernel's chain CTA: the compute warps and the sync warp
__device__ __forceinline__ void bar_chain() { asm volatile("bar.sync 2, %0;" ::"n"(NCT + 32) : "memory"); }
using wn::pack_h2;
using wn::unpack_h2;
__device__ __forceinline__ uint32_t u32(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }
__device__ __forceinline__ __half2 h2(uint32_t v) { return *reinterpret_cast<__half2*>(&v); }

__device__ __forceinline__ void cp_async4(uint32_t dst, const void* src) { asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory"); }
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory"); }
// the mbarrier receives one arrival once every cp.async this thread has issued so far has landed
__device__ __forceinline__ void cp_async_arrive_noinc(uint32_t bar) { asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait_pending() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ------------------------------------------------------------------------------------------------ layouts
__host__ __device__ inline int lat_tiles(int B) { return (B + TU - 1) / TU; }

// The latency layouts for wn_layout.cuh, both per 16-utterance tile of the engine's batch; a unit is one 4-byte word of a channel
// pair (c, c + 1), c even, of one utterance row b: tile b / 16, row r = b mod 16, g = r mod 8.
struct LatLayout {
    using TD = __half;
    static constexpr int STORE_UNIT = 2, RING_UNIT = 2;
    // Conditioning: fp16, [N][L][tiles][8 warps][32 lanes][16 B]: the uint4 of thread (w, lane = 4 g + t) holds, as half2 pairs of
    // channels (c, c+1), c = 8 w + 2 t:  .x = (row g, tanh c) .y = (row g+8, tanh c) .z = (row g, sigmoid R+c) .w = (row g+8, sigmoid R+c)
    // i.e. exactly the accumulator fragment the thread adds it to.  Unit k is channels (2k, 2k + 1) of the 2R; k >= 32: sigmoid.
    static __device__ WnVec<__half, 2>* store_unit(const WnConfig& c, void* store, size_t sl, int b, int k)
    {
        const int tile = b / TU, r = b % TU, g = r & 7, hi = r >> 3, sig = k >> 5, w = (k & 31) >> 2, t = k & 3;
        return reinterpret_cast<WnVec<__half, 2>*>(static_cast<unsigned char*>(store) + (sl * lat_tiles(c.B) + tile) * 4096 +
                                                   (size_t)(w * 32 + g * 4 + t) * 16 + (size_t)(2 * sig + hi) * 4);
    }
    // The history ring: per entry (slot x L + layer) one 2 KB image per tile.  Row r of a tile is the 32 words that store_x and the
    // embedding store write for it: channels (c, c + 1) = (2k, 2k + 1) sit at k-step j = c / 16, lane 4 g + (c mod 8) / 2, word
    // 2 ((c / 8) mod 2) + (r >= 8) of the lane's 16-byte group.
    static __device__ WnVec<__half, 2>* ring_unit(const WnConfig& c, void* ring, size_t e, int, int b, int k)
    {
        const int tile = b / TU, r = b % TU, g = r & 7, hi = r >> 3, j = k >> 3, half = (k >> 2) & 1, t = k & 3;
        return reinterpret_cast<WnVec<__half, 2>*>(static_cast<unsigned char*>(ring) + (e * lat_tiles(c.B) + tile) * 2048 + (size_t)j * 512 +
                                                   (size_t)(4 * g + t) * 16 + (size_t)(2 * half + hi) * 4);
    }
    static size_t store_bytes(const WnConfig& c) { return (size_t)c.N * c.L * lat_tiles(c.B) * 4096; }
    static size_t ring_bytes(const WnConfig& c) { return (size_t)(c.maxDil + 1) * c.L * lat_tiles(c.B) * 2048; }
};

// The whole store, one thread per 16-byte group of the layout: rows g and g + 8 and both gate halves in one store, and zero rows
// past the batch.  The per-row wn_convert_rows would store the same bytes as four 4-byte words and leave the padding rows alone.
__global__ void lat_cond_kernel(size_t total, WnConfig cfg, unsigned char* __restrict__ dst, const float* __restrict__ src, int first_sample)
{
    const int ntiles = lat_tiles(cfg.B);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int th = (int)(i & 255), w = th >> 5, lane = th & 31, g = lane >> 2, t = lane & 3;
        const size_t slt = i >> 8;                       // (s * L + l) * ntiles + tile
        const int tile = (int)(slt % ntiles);
        const size_t sl = slt / ntiles;                  // s * L + l
        const int c = 8 * w + 2 * t;
        uint32_t o[4] = {0, 0, 0, 0};
#pragma unroll
        for (int hi = 0; hi < 2; hi++) {
            const int b = tile * TU + g + 8 * hi;
            if (b < cfg.B) {
                const float* row = src + (sl * cfg.B + b) * 128;
                const float2 ft = *reinterpret_cast<const float2*>(row + c), fs = *reinterpret_cast<const float2*>(row + 64 + c);
                __half2 a = __floats2half2_rn(ft.x, ft.y), s = __floats2half2_rn(fs.x, fs.y);
                o[hi] = *reinterpret_cast<uint32_t*>(&a);
                o[2 + hi] = *reinterpret_cast<uint32_t*>(&s);
            }
        }
        // the group starts at the unit of (row g, tanh c)
        *reinterpret_cast<uint4*>(LatLayout::store_unit(cfg, dst, (size_t)first_sample * cfg.L + sl, tile * TU + g, c / 2)) = make_uint4(o[0], o[1], o[2], o[3]);
    }
}

// ------------------------------------------------------------------------------------------------ pack
// blob (fp16, column-major M x K matrices as uploaded) -> weight image in mma.m16n8k16 B-fragment order.
// Element (n-tile nt, k-step pair jp, lane = 4 g + t) of a matrix W[M][K] is the uint4
//   { W[8nt+g][32jp+2t .. +1], W[8nt+g][32jp+8+2t ..], W[8nt+g][32jp+16+2t ..], W[8nt+g][32jp+24+2t ..] }
// = (b0, b1) of k-step 2jp and (b0, b1) of k-step 2jp+1.
__device__ __forceinline__ void frag_pos(int row, int k, int njp, size_t& byte_off)
{
    const int nt = row >> 3, g = row & 7, jp = k >> 5, kk = k & 31, comp = kk >> 3, t = (kk & 7) >> 1, e = kk & 1;
    byte_off = ((size_t)(nt * njp + jp) * 32 + (g * 4 + t)) * 16 + comp * 4 + e * 2;
}
__global__ void lat_pack_kernel(WnParams p, unsigned char* __restrict__ img, LatImage im)
{
    const int S = p.S, L = p.L;
    const __half* Wprev = static_cast<const __half*>(p.Wprev);
    const __half* Wcur = static_cast<const __half*>(p.Wcur);
    const __half* Wres = static_cast<const __half*>(p.Wres);
    const __half* Wskip = static_cast<const __half*>(p.Wskip);
    const __half* Wzs = static_cast<const __half*>(p.Wzs);
    const __half* Wza = static_cast<const __half*>(p.Wza);
    const size_t gstride = (size_t)gridDim.x * blockDim.x;
    const size_t g0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    auto put = [&](size_t base, int row, int k, int njp, __half v) {
        size_t o;
        frag_pos(row, k, njp, o);
        *reinterpret_cast<__half*>(img + base + o) = v;
    };
    for (size_t i = g0; i < (size_t)L * 128 * 64; i += gstride) {
        const int l = (int)(i / (128 * 64)), c = (int)(i % (128 * 64)) / 64, k = (int)(i % 64);
        const size_t lb = (size_t)l * im.layer_bytes;
        put(lb, c, k, 2, Wcur[(size_t)l * 128 * 64 + c + (size_t)k * 128]);
        put((size_t)((l + L - 1) % L) * im.layer_bytes + 16384, c, k, 2, Wprev[(size_t)l * 128 * 64 + c + (size_t)k * 128]);   // rides with the layer before it
        if (c < 64) put(lb + 32768, c, k, 2, Wres[(size_t)l * 64 * 64 + c + (size_t)k * 64]);
    }
    for (size_t i = g0; i < (size_t)L * S * 64; i += gstride) {
        const int l = (int)(i / ((size_t)S * 64)), s = (int)((i / 64) % S), k = (int)(i % 64);
        put((size_t)l * im.layer_bytes + 40960, s, k, 2, Wskip[(size_t)l * S * 64 + s + (size_t)k * S]);
    }
    // output matrices: ring piece q holds k-step pairs [q OJP, (q+1) OJP) of all 32 n-tiles
    {
        const int ojp = S / 128;
        const size_t piece = (size_t)32 * ojp * 512;
        for (size_t i = g0; i < (size_t)A * S; i += gstride) {
            const int a = (int)(i / S), s = (int)(i % S);
            const int jp = s >> 5, q = jp / ojp;
            put(im.off_zs + (size_t)q * piece, a, (s & 31) + 32 * (jp % ojp), ojp, Wzs[a + (size_t)s * A]);
        }
    }
    {
        const int ojp = A / 128;
        const size_t piece = (size_t)32 * ojp * 512;
        for (size_t i = g0; i < (size_t)A * A; i += gstride) {
            const int a = (int)(i / A), z = (int)(i % A);
            const int jp = z >> 5, q = jp / ojp;
            put(im.off_za + (size_t)q * piece, a, (z & 31) + 32 * (jp % ojp), ojp, Wza[a + (size_t)z * A]);
        }
    }
    float* bias = reinterpret_cast<float*>(img + im.off_bias);
    const __half* Bh = static_cast<const __half*>(p.Bh);
    const __half* Bres = static_cast<const __half*>(p.Bres);
    const __half* Bskip = static_cast<const __half*>(p.Bskip);
    for (size_t i = g0; i < (size_t)L * 256; i += gstride) {
        const int l = (int)(i / 256), w = (int)(i % 256) / 32, t = (int)(i % 32) / 8, e = (int)(i % 8);
        const int c = 8 * w + 2 * t + (e & 1);
        float v = 0.f;
        if (e < 2) v = __half2float(Bh[(size_t)l * 128 + c]);
        else if (e < 4) v = __half2float(Bh[(size_t)l * 128 + 64 + c]);
        else if (e < 6) v = __half2float(Bres[(size_t)l * 64 + c]);
        bias[im.b_layer + i] = v;
    }
    for (size_t s = g0; s < (size_t)S; s += gstride) {
        float acc = 0.f;
        for (int l = 0; l < L; l++) { acc += __half2float(Bskip[(size_t)l * S + s]); bias[im.b_skpre + (size_t)l * S + s] = acc; }
    }
    for (size_t i = g0; i < (size_t)A; i += gstride) {
        bias[im.b_bzs + i] = __half2float(static_cast<const __half*>(p.Bzs)[i]);
        bias[im.b_bza + i] = __half2float(static_cast<const __half*>(p.Bza)[i]);
    }
}

// ------------------------------------------------------------------------------------------------ stages of both latency kernels
// Each stage is called by both wn_lat_kernel and wn_lat2_kernel.  Per thread of the eight compute warps: warp w, lane = 4 g + t4;
// the thread holds rows g and g + 8 of the 16 utterances and channels 8 w + 2 t4 + {0, 1} of an activation tile (k-step w >> 1,
// half w & 1 of its A fragments).  The cluster kernel also runs tiles of TR = 8 utterances: the MMA is still m16n8k16, rows 8-15
// of every A fragment are the constant 0 and the epilogue of accumulator rows g + 8 is skipped.  Rows 0-7 go through the same
// HMMAs in the same order, so every value they produce is the one a 16-row tile produces.
struct StepIt { int t, l, slot; };       // coordinates of a layer step: sample, layer, history-ring slot of that sample

// An activation tile in shared memory (TR rows x 64 channels, fp16) is kept in A-fragment order, TR bytes per lane and k-step:
// 16 rows = the whole fragment (a0 a1 a2 a3), 8 rows = only the words of rows g (a0 a2).  The thread's slot of channels
// 8 w + 2 t4 + {0, 1}: k-step w >> 1, half w & 1.
template <int TR> __device__ __forceinline__ uint32_t xslot(int w, int lane)
{
    return (uint32_t)((w >> 1) * 32 * TR + lane * TR + (w & 1) * (TR / 2));
}
// A fragment of k-step j of such a tile
template <int TR> __device__ __forceinline__ void load_a_rows(uint32_t (&a)[4], uint32_t tile, int j, int lane)
{
    if (TR == TU) load_a(a, tile + (uint32_t)(j * 512 + lane * 16));
    else { const uint2 v = lds64(tile + (uint32_t)(j * 256 + lane * 8)); a[0] = v.x; a[1] = 0u; a[2] = v.y; a[3] = 0u; }
}

// this tile's rows of a 16-byte group of a 16-row layout (words: row g, row g + 8, row g, row g + 8 of two k or channel halves):
// the whole group for 16 rows; for 8 rows, half `hi` of the 16-row tile, as (row g word, 0, row g word, 0)
template <int TR> __device__ __forceinline__ uint4 own_rows(uint4 v, bool hi)
{
    if (TR == TU) return v;
    return make_uint4(hi ? v.y : v.x, 0u, hi ? v.w : v.z, 0u);
}

// byte offset of history-ring row `row` (= slot x L + layer) of `rstride` bytes.  A ring of at most 4 GiB runs the kernels' WIDE = false
// instantiations: every row starts below 2^32 bytes, so the 32-bit product is exact, and it is the form the step loop is fastest
// with (the 64-bit forms tried measured 0.5-6 % slower at C3, B = 64, H100 80GB HBM3 at 700 W).  A larger ring (C3 from 3 265
// utterances, L64 maxDil 2048 from 256) runs WIDE = true, whose offsets are 64-bit.
template <bool WIDE> __device__ __forceinline__ size_t ring_off(uint32_t row, uint32_t rstride)
{
    return WIDE ? (size_t)row * rstride : (size_t)(row * rstride);
}
// WIDE for a ring of `ntiles` tiles per entry (LatLayout::ring_bytes) past 4 GiB
static bool lat_ring_wide(int maxDil, int L, int ntiles) { return (size_t)(maxDil + 1) * L * ntiles * 2048 > ((size_t)1 << 32); }

// feedback state of the tile ([TR] current index, [TR] previous index) of utterances ub .. ub + TR - 1 -> yCur / yPrev
template <int TR = TU>
__device__ __forceinline__ void store_ys(const WnParams& p, int B, const int* ys, int ub, int tid)
{
    if (tid < TR && ub + tid < B) { p.yCur[ub + tid] = ys[tid]; p.yPrev[ub + tid] = ys[TR + tid]; }
}
// this thread's values of x (fp16) -> the x exchange tile and row `row` (= history slot x L + layer) of the history ring.  The
// ring keeps the 16-row A-fragment order; an 8-row tile writes only its rows' words (`gring` points at them).
template <int TR = TU, bool WIDE = false>
__device__ __forceinline__ void store_x(const float (&x)[4], uint32_t xtile, unsigned char* gring, uint32_t row, uint32_t rstride, int w)
{
    unsigned char* gp = gring + ring_off<WIDE>(row, rstride) + (w >> 1) * 512 + (w & 1) * 8;
    const uint32_t x01 = pack_h2(x[0], x[1]);
    if (TR == TU) {
        const uint32_t x23 = pack_h2(x[2], x[3]);
        sts64(xtile, x01, x23);
        stg_v2(gp, x01, x23);
    } else {
        sts32(xtile, x01);
        stg_b32(gp, x01);
    }
}
// B fragments of warp w's gate columns for a K = 64 GEMM: tanh and sigmoid n-tiles, k-step pairs 0 and 1
struct GateW { uint4 t0, g0, t1, g1; };
__device__ __forceinline__ GateW lds_gate_w(uint32_t piece, uint32_t o_t0, uint32_t o_g0)
{
    return {lds128(piece + o_t0), lds128(piece + o_g0), lds128(piece + o_t0 + 512), lds128(piece + o_g0 + 512)};
}
// K = 64 gate GEMM (Wcur.x or Wprev.x[t-d]) as two independent chains: k-steps 0-1 into d, 2-3 into u ([0] tanh, [1] sigmoid)
__device__ __forceinline__ void hmma_k64(float (&d)[2][4], float (&u)[2][4], const uint32_t (&a)[4][4], const GateW& b)
{
    hmma(d[0], a[0], b.t0.x, b.t0.y); hmma(d[1], a[0], b.g0.x, b.g0.y); hmma(u[0], a[2], b.t1.x, b.t1.y); hmma(u[1], a[2], b.g1.x, b.g1.y);
    hmma(d[0], a[1], b.t0.z, b.t0.w); hmma(d[1], a[1], b.g0.z, b.g0.w); hmma(u[0], a[3], b.t1.z, b.t1.w); hmma(u[1], a[3], b.g1.z, b.g1.w);
}
__device__ __forceinline__ void gemm_k64(float (&d)[2][4], const uint32_t (&a)[4][4], const GateW& b)
{
    float u[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
    hmma_k64(d, u, a, b);
#pragma unroll
    for (int i = 0; i < 4; i++) { d[0][i] += u[0][i]; d[1][i] += u[1][i]; }
}
// h = tanh(a[:R]) * sigmoid(a[R:]) in packed fp16 (MUFU; sigmoid(x) = 0.5 tanh(x/2) + 0.5) -> the h tile; returns the two words
// (8-row tiles: row g only, h23 = 0)
template <int TR = TU>
__device__ __forceinline__ void gate(const float (&a)[2][4], uint32_t htile, uint32_t& h01, uint32_t& h23)
{
    const __half2 half = __floats2half2_rn(0.5f, 0.5f);
    const __half2 tg0 = wn::tanh_h2(h2(pack_h2(a[0][0], a[0][1])));
    const __half2 sg0 = __hfma2(wn::tanh_h2(h2(pack_h2(0.5f * a[1][0], 0.5f * a[1][1]))), half, half);
    h01 = u32(__hmul2(tg0, sg0));
    if (TR == TU) {
        const __half2 tg1 = wn::tanh_h2(h2(pack_h2(a[0][2], a[0][3])));
        const __half2 sg1 = __hfma2(wn::tanh_h2(h2(pack_h2(0.5f * a[1][2], 0.5f * a[1][3]))), half, half);
        h23 = u32(__hmul2(tg1, sg1));
        sts64(htile, h01, h23);
    } else {
        h23 = 0u;
        sts32(htile, h01);
    }
}
// Wres.h as two half-K chains (B fragments bw0, bw1 of k-step pairs 0 and 1)
__device__ __forceinline__ void hmma_res(float (&ra)[4], float (&rb)[4], const uint32_t (&ha)[4][4], uint4 bw0, uint4 bw1)
{
    hmma(ra, ha[0], bw0.x, bw0.y); hmma(rb, ha[2], bw1.x, bw1.y);
    hmma(ra, ha[1], bw0.z, bw0.w); hmma(rb, ha[3], bw1.z, bw1.w);
}
// x' = ((ra + rb) + Bres) + x; below the last layer x' goes to the x tile and history ring row `row` (8-row tiles: row g only)
template <int TR = TU, bool WIDE = false>
__device__ __forceinline__ void residual(float (&x)[4], const float (&ra)[4], const float (&rb)[4], float2 br, bool store, uint32_t xtile,
                                         unsigned char* gring, uint32_t row, uint32_t rstride, int w)
{
    x[0] = ((ra[0] + rb[0]) + br.x) + x[0]; x[1] = ((ra[1] + rb[1]) + br.y) + x[1];
    if (TR == TU) { x[2] = ((ra[2] + rb[2]) + br.x) + x[2]; x[3] = ((ra[3] + rb[3]) + br.y) + x[3]; }
    if (store) store_x<TR, WIDE>(x, xtile, gring, row, rstride, w);
}
template <bool DUMP>
__device__ __forceinline__ void dump_xt(const WnParams& p, int B, int l, int b0, int b1, int cw, const float (&x)[4])
{
    if (DUMP) {
        if (b0 < B) { p.xtOut[((size_t)l * B + b0) * R + cw] = x[0]; p.xtOut[((size_t)l * B + b0) * R + cw + 1] = x[1]; }
        if (b1 < B) { p.xtOut[((size_t)l * B + b1) * R + cw] = x[2]; p.xtOut[((size_t)l * B + b1) * R + cw + 1] = x[3]; }
    }
}
// relu(skip + Bskip) of one skip n-tile (columns c, c + 1), packed as A-fragment words of rows g and g + 8; the sum restarts at 0
__device__ __forceinline__ void relu_skip(float (&sk)[4], const float* bskip, int c, uint32_t& lo, uint32_t& hi)
{
    const float b0f = bskip[c], b1f = bskip[c + 1];
    lo = pack_h2(fmaxf(sk[0] + b0f, 0.f), fmaxf(sk[1] + b1f, 0.f));
    hi = pack_h2(fmaxf(sk[2] + b0f, 0.f), fmaxf(sk[3] + b1f, 0.f));
    sk[0] = sk[1] = sk[2] = sk[3] = 0.f;
}


// ------------------------------------------------------------------------------------------------ the kernel

// What both roles of wn_lat_kernel (the TMA producer lane and the compute warps) use; set once, by the kernel's prologue.
struct LatCta {
    const WnParams& p;
    const unsigned char* img;                   // the tile's weight image and previous-index embedding table (its model's)
    const void* embPrev;
    LatImage im;
    uint32_t sm;                                // shared-memory base
    int L, B, tid, w, lane, tile, slots, t_begin, t_end;
    const float* gbias;
    uint32_t s_full, s_empty, s_pfull;          // mbarriers: Cfg::B_*
    int* dil;
    int* ys;                                    // [TU] current index, [TU] previous index
    float* s_bout;
    // debug timeline: role 0 = compute thread 0, role 2 = producer; words (tag << 48 | clock)
    unsigned long long* trc;
    int tr_t;
};
#define TRACE(role, tag) do { if (TRC && trc && t == tr_t && trn < 1023) trc[(role) * 1024 + trn++] = ((unsigned long long)(tag) << 48) | (clock64() & 0xFFFFFFFFFFFFull); } while (0)

// TMA producer (one lane): the pieces in consumption order, each refilled as soon as ITS previous occupant has been consumed (two
// layers of lead for every piece)
template <int S, bool TRC>
__device__ __forceinline__ void lat_producer(const LatCta& c, int& trn)
{
    using C = Cfg<S>;
    const unsigned char* img = c.img;
    const LatImage& im = c.im;
    const uint32_t sm = c.sm, s_full = c.s_full, s_empty = c.s_empty;
    const int L = c.L, t_begin = c.t_begin, t_end = c.t_end;
    unsigned long long* trc = c.trc;
    const int tr_t = c.tr_t;
    uint32_t pc = 0;
    auto put = [&](const unsigned char* src, uint32_t bytes) {
        const uint32_t idx = (pc >> 1) & 1, bo = C::ring_bar(pc & 1, idx);
        const uint32_t dst = (pc & 1) ? sm + C::O_RING2 + idx * C::SLOT2 : sm + C::O_RING1 + idx * C::SLOT1;
        mbar_wait(s_empty + bo, ((pc / C::NSLOT) & 1) ^ 1);
        mbar_arrive_expect_tx(s_full + bo, bytes);
        tma_load_1d(dst, src, bytes, s_full + bo);
        pc++;
    };
    for (int t = t_begin; t < t_end; t++) {
        for (int l = 0; l < L; l++) {
            const unsigned char* src = img + (size_t)l * im.layer_bytes;
            put(src, C::P1_BYTES);
            put(src + C::P1_BYTES, C::P2_BYTES);
            TRACE(2, 100 + l);
        }
        for (int q = 0; q < C::NQ; q++) {
            put(q < C::NQ_ZS ? img + im.off_zs + (size_t)q * C::ZS_PIECE : img + im.off_za + (size_t)(q - C::NQ_ZS) * C::ZA_PIECE,
                q < C::NQ_ZS ? C::ZS_PIECE : C::ZA_PIECE);
            TRACE(2, 200 + q);
        }
    }
}

// the eight compute warps
template <int S, bool DUMP, bool TRC, bool WIDE>
__device__ __forceinline__ void lat_compute(const LatCta& c, int& trn, const int ntiles_alloc)
{
    using C = Cfg<S>;
    const WnParams& p = c.p;
    const unsigned char* img = c.img;
    const LatImage& im = c.im;
    const uint32_t sm = c.sm, s_full = c.s_full, s_empty = c.s_empty, s_pfull = c.s_pfull;
    const int L = c.L, B = c.B, tid = c.tid, lane = c.lane, tile = c.tile, slots = c.slots, t_begin = c.t_begin, t_end = c.t_end;
    const float* gbias = c.gbias;
    const int* dil = c.dil;
    int* ys = c.ys;
    const float* s_bout = c.s_bout;
    unsigned long long* trc = c.trc;
    const int tr_t = c.tr_t;
    const int w = c.w, g = lane >> 2, t4 = lane & 3;
    const int b0 = tile * TU + g, b1 = b0 + 8;
    const bool v0 = b0 < B, v1 = b1 < B;
    const uint32_t cstride = (uint32_t)ntiles_alloc * 4096u, rstride = (uint32_t)ntiles_alloc * 2048u;
    const unsigned char* gcond = static_cast<const unsigned char*>(p.Lh) + (size_t)tile * 4096 + (size_t)(w * 32 + lane) * 16;
    unsigned char* gring = static_cast<unsigned char*>(p.ring) + (size_t)tile * 2048 + (size_t)lane * 16;
    const float* gbl = gbias + im.b_layer + (size_t)(w * 4 + t4) * 8;
    const int jw = w >> 1, hw = w & 1;             // this warp's 8 channels = k-step jw, half hw of an activation tile
    const uint32_t lane16 = (uint32_t)lane * 16;
    const uint32_t xchg = (uint32_t)(jw * 512 + hw * 8) + lane16;
    const int cw = 8 * w + 2 * t4;                 // first of the thread's two channels inside the warp's slice
    // this thread's B-fragment offsets inside the ring pieces
    const uint32_t o_t0 = (uint32_t)(w * 2) * 512 + lane16, o_g0 = (uint32_t)((8 + w) * 2) * 512 + lane16;   // + 512 for the second k-step pair
    const uint32_t o_res = (uint32_t)(w * 2) * 512 + lane16, o_skip = 8192u + (uint32_t)(w * C::NSK * 2) * 512 + lane16;
    const uint32_t o_out = (uint32_t)(4 * w) * 512;                                                         // output pieces: x OJP, + lane16

    auto advance = [&](StepIt& it) { if (++it.l == L) { it.l = 0; it.t++; if (++it.slot == slots) it.slot = 0; } };
    auto release = [&](uint32_t bar) { __syncwarp(); if (lane == 0) mbar_arrive(bar); };
    // Every mbarrier wait costs ~90 cycles even when the phase completed long ago (TRYWAIT latency).  The barriers of the coming
    // step are therefore looked at once, at the end of the running step (measured: 40.1 kHz at C3 B=64 against 38.4 kHz with
    // plain waits at the point of use, and 35.9 kHz with blocking waits moved behind the preceding HMMA batches).
    auto probe = [&](uint32_t bar, uint32_t parity) -> bool { return mbar_try_wait(bar, parity); };
    auto ensure = [&](bool ok, uint32_t bar, uint32_t parity) { if (!ok) mbar_wait(bar, parity); };

    // dilated history x_l[t - d] (zero before the start of the utterance, nv_wavenet.cuh:106) of the step `itp`: staged three
    // steps ahead into a 3-slot shared-memory ring by warps 0-3 (128 threads x 16 B, cp.async; completion on an mbarrier).
    // itp.t counts the (clamped) absolute time of the WnParams, so the test against d is the utterance's.
    StepIt itp{p.hist_t, 0, p.ring_slot};
    const int h_end = p.hist_t + p.count;
    uint32_t pcnt = 0;                             // tiles staged so far (slot = pcnt % NPST)
    auto stage_history = [&]() {
        if (w < 4) {
            const uint32_t slot3 = pcnt % C::NPST;
            const int d = dil[itp.l];
            const uint32_t dst = sm + C::O_PST + slot3 * 2048 + (uint32_t)(w * 32 + lane) * 16;
            if (itp.t >= h_end || itp.t < d) {
                sts128(dst, make_uint4(0, 0, 0, 0));
                mbar_arrive(s_pfull + 8 * slot3);
            } else {
                int sl = itp.slot - d; if (sl < 0) sl += slots;
                cp_async16(dst, gring - lane16 + ring_off<WIDE>(sl * L + itp.l, rstride) + (size_t)(w * 32 + lane) * 16);
                cp_async_arrive_noinc(s_pfull + 8 * slot3);
            }
        }
        pcnt++;
        advance(itp);
    };

    uint32_t xa[4][4];
    uint4 cbA = make_uint4(0, 0, 0, 0), cbB = make_uint4(0, 0, 0, 0);
    float accp[2][4];                              // pre-activation of the coming step: Wprev.x[t-d] + Bh + Lh
    float2 brn;                                    // Bres pair of the coming step
    float4 bh_next = make_float4(0.f, 0.f, 0.f, 0.f); float2 br_next = make_float2(0.f, 0.f);            // Bh / Bres pairs of the step after (prefetched a layer ahead)
    float xres[4] = {0.f, 0.f, 0.f, 0.f};
    float sk[C::NSK][4];
#pragma unroll
    for (int i = 0; i < C::NSK; i++) sk[i][0] = sk[i][1] = sk[i][2] = sk[i][3] = 0.f;
    const unsigned char* cptr = gcond + (size_t)t_begin * L * cstride;      // conditioning of step it3 (steps are consecutive in memory)

    // accp <- (Bh + Lh) + Wprev . x[t-d] for the coming step `it1` (its staged history tile is number `pn`, its conditioning
    // sits in cbA / cbB by parity); Wprev rides in the SAME ring piece as the current layer's Wcur (`p1`; the very first
    // one comes from global memory).  Then the conditioning of step it3 is fetched.  Independent of the current layer's data.
    StepIt it1{0, 0, 0}, it3{0, 0, 0};
    uint32_t pn = 0, kp = 0;                       // kp = parity of the running step
    auto prep = [&](const uint32_t p1, const bool from_global, const bool pf_ok) {
        brn = br_next;
        const uint4 cb = kp ? cbA : cbB;           // step k consumes the buffer of parity (k + 1) & 1 ...
        {
            const float2 c0 = unpack_h2(cb.x), c1 = unpack_h2(cb.y), c2 = unpack_h2(cb.z), c3 = unpack_h2(cb.w);
            accp[0][0] = bh_next.x + c0.x; accp[0][1] = bh_next.y + c0.y; accp[0][2] = bh_next.x + c1.x; accp[0][3] = bh_next.y + c1.y;
            accp[1][0] = bh_next.z + c2.x; accp[1][1] = bh_next.w + c2.y; accp[1][2] = bh_next.z + c3.x; accp[1][3] = bh_next.w + c3.y;
        }
        const uint32_t slot3 = pn % C::NPST;
        if (it1.t < t_end) {
            GateW bw;
            if (from_global) {
                const unsigned char* gp = img + (size_t)(L - 1) * im.layer_bytes + C::W_PREV;
                bw = {ldg_nc_v4(gp + o_t0), ldg_nc_v4(gp + o_g0), ldg_nc_v4(gp + o_t0 + 512), ldg_nc_v4(gp + o_g0 + 512)};
            } else {
                bw = lds_gate_w(p1 + C::W_PREV, o_t0, o_g0);
            }
            ensure(pf_ok, s_pfull + 8 * slot3, (pn / C::NPST) & 1);
            uint32_t pb[4][4];
#pragma unroll
            for (int j = 0; j < 4; j++) load_a(pb[j], sm + C::O_PST + slot3 * 2048 + j * 512 + lane16);
            gemm_k64(accp, pb, bw);
        }
        pn++;
        {   // ... and refills it with the conditioning of step k + 3
            const unsigned char* src = cptr;
            cptr += cstride;
            const bool live = it3.t < t_end;       // past the end the stale value is never used (the prep of such a step is skipped)
            ldg_nc_v4_if(cbA, src, live && kp != 0);
            ldg_nc_v4_if(cbB, src, live && kp == 0);
        }
        advance(it1); advance(it3);
        bh_next = *reinterpret_cast<const float4*>(gbl + it1.l * 256);
        br_next = *reinterpret_cast<const float2*>(gbl + it1.l * 256 + 4);
    };

    // ---------------- prologue: previous-index rows of the first sample, prefetch pipeline
    {
        const uint32_t* ep = static_cast<const uint32_t*>(c.embPrev);
        sts32(sm + C::O_EPBUF + (g * EROW + 4 * w + t4) * 4, ep[ys[TU + g] * 32 + 4 * w + t4]);
        sts32(sm + C::O_EPBUF + ((g + 8) * EROW + 4 * w + t4) * 4, ep[ys[TU + g + 8] * 32 + 4 * w + t4]);
    }
    StepIt it0{t_begin, 0, p.ring_slot};
    stage_history(); stage_history(); stage_history();              // history tiles of steps 0, 1, 2
    {
        it1 = it0; it3 = it0;
        kp = 1;                                                     // the prologue plays "step -1": consumes cbA (step 0), refills it with step 2
        cbA = ldg_nc_v4(cptr); cptr += cstride;
        { StepIt i1 = it0; advance(i1); cbB = i1.t < t_end ? ldg_nc_v4(cptr) : make_uint4(0, 0, 0, 0); cptr += cstride; }
        advance(it3); advance(it3);
        bh_next = *reinterpret_cast<const float4*>(gbl); br_next = *reinterpret_cast<const float2*>(gbl + 4);
        prep(0, true, false);                                       // leaves it1 = step 1, it3 = step 3
        kp = 0;
    }
    bar_compute();

    // ring bookkeeping: a layer step uses slot `sb` of both piece types; the parity of its barriers is `fph`
    uint32_t sb = 0, fph = 0;

    bool ok_f1 = false, ok_f2 = false, ok_pf = false;          // what the look at the coming step's barriers returned
    // one layer step
    auto step = [&](const int t, const int l) {
        const uint32_t p1 = sm + C::O_RING1 + sb * C::SLOT1, p2 = sm + C::O_RING2 + sb * C::SLOT2;
        const uint32_t f1 = s_full + C::ring_bar(0, sb), f2 = s_full + C::ring_bar(1, sb), e1 = s_empty + C::ring_bar(0, sb), e2 = s_empty + C::ring_bar(1, sb);
        const float2 br = brn;
        // ---- a = Wcur.x + [Wprev.x[t-d] + Bh + Lh]   (nv_wavenet.cuh:131-157); the two halves of K as independent chains
        ensure(ok_f1, f1, fph);
        gemm_k64(accp, xa, lds_gate_w(p1, o_t0, o_g0));
        // ---- h = tanh(a[:R]) * sigmoid(a[R:])
        {
            uint32_t h01, h23;
            gate(accp, sm + C::O_HBUF + xchg, h01, h23);
        }
        if (tid == 0) TRACE(0, 12);
        // ---- while the other warps finish their part of h: the dilated-history half of the next step's pre-activation
        // (after the last layer: layer 0 of the next sample); then this piece of the ring is free
        prep(p1, false, ok_pf);
        release(e1);
        bar_compute();
        uint32_t ha[4][4];
#pragma unroll
        for (int j = 0; j < 4; j++) load_a(ha[j], sm + C::O_HBUF + j * 512 + lane16);
        if (tid == 0) TRACE(0, 10);
        // ---- x' = Wres.h + Bres + x   (nv_wavenet.cuh:185-207); two half-K chains
        float ra[4] = {0.f, 0.f, 0.f, 0.f}, rb[4] = {0.f, 0.f, 0.f, 0.f};
        ensure(ok_f2, f2, fph);
        {
            const uint4 bw0 = lds128(p2 + o_res), bw1 = lds128(p2 + o_res + 512);
            hmma_res(ra, rb, ha, bw0, bw1);
        }
        residual<TU, WIDE>(xres, ra, rb, br, l + 1 < L, sm + C::O_XBUF + xchg, gring, (uint32_t)(it0.slot * L + l + 1), rstride, w);
        if (tid == 0) TRACE(0, 14);
        dump_xt<DUMP>(p, B, l, b0, b1, cw, xres);
        // ---- while the other warps finish their part of x': skip += Wskip.h   (biases are added once, after the last layer)
#pragma unroll
        for (int jp = 0; jp < 2; jp++) {
            uint4 bw[C::NSK];
#pragma unroll
            for (int i = 0; i < C::NSK; i++) bw[i] = lds128(p2 + o_skip + (i * 2 + jp) * 512);
#pragma unroll
            for (int i = 0; i < C::NSK; i++) hmma(sk[i], ha[2 * jp], bw[i].x, bw[i].y);
#pragma unroll
            for (int i = 0; i < C::NSK; i++) hmma(sk[i], ha[2 * jp + 1], bw[i].z, bw[i].w);
        }
        release(e2);
        stage_history();                           // the history tile of three steps ahead
        {   // look at the coming step's barriers now; the answers are consumed a barrier later
            const uint32_t nsb = sb ^ 1, nph = fph ^ sb;
            mbar_try_wait3(s_full + C::ring_bar(0, nsb), nph, s_full + C::ring_bar(1, nsb), nph, s_pfull + 8 * (pn % C::NPST), (pn / C::NPST) & 1, ok_f1, ok_f2, ok_pf);
        }
        if (tid == 0) TRACE(0, 15);
        if (DUMP) {
            const float* pre = gbias + im.b_skpre + (size_t)l * S;
#pragma unroll
            for (int i = 0; i < C::NSK; i++) {
                const int c = 8 * (w * C::NSK + i) + 2 * t4;
                float o0 = sk[i][0] + pre[c], o1 = sk[i][1] + pre[c + 1], o2 = sk[i][2] + pre[c], o3 = sk[i][3] + pre[c + 1];
                if (l == L - 1) { o0 = fmaxf(o0, 0.f); o1 = fmaxf(o1, 0.f); o2 = fmaxf(o2, 0.f); o3 = fmaxf(o3, 0.f); }
                if (v0) { p.skipOut[((size_t)l * B + b0) * S + c] = o0; p.skipOut[((size_t)l * B + b0) * S + c + 1] = o1; }
                if (v1) { p.skipOut[((size_t)l * B + b1) * S + c] = o2; p.skipOut[((size_t)l * B + b1) * S + c + 1] = o3; }
            }
        }
        if (l + 1 < L) {
            bar_compute();
#pragma unroll
            for (int j = 0; j < 4; j++) load_a(xa[j], sm + C::O_XBUF + j * 512 + lane16);
        }
        if (tid == 0) TRACE(0, 11);
        fph ^= sb; sb ^= 1; kp ^= 1;               // slot alternates every step, barrier parity every second step
    };

    uint32_t epar = 0;                             // parity of the sample (epbuf buffer)
    for (int t = t_begin; t < t_end; t++) {
        // ---------------- embedding (reference.cpp:42-57): x0 = [tanh](embPrev[yPrev] + embCur[yCur]), this warp's 8 channels
        if (tid == 0) TRACE(0, 1);
        const float sel0 = (2 * w + 0 + tile * TU) < B ? p.sel[(size_t)t * B + tile * TU + 2 * w] : 0.5f;
        const float sel1 = (2 * w + 1 + tile * TU) < B ? p.sel[(size_t)t * B + tile * TU + 2 * w + 1] : 0.5f;
        {
            const int yc0 = ys[g], yc1 = ys[g + 8];
            const uint32_t eo = sm + C::O_EPBUF + epar * (TU * EROW * 4);
            const float2 a0 = unpack_h2(lds32(eo + (g * EROW + 4 * w + t4) * 4)), a1 = unpack_h2(lds32(eo + ((g + 8) * EROW + 4 * w + t4) * 4));
            const float2 c0 = unpack_h2(lds32(sm + C::O_EMB + (yc0 * EROW + 4 * w + t4) * 4)), c1 = unpack_h2(lds32(sm + C::O_EMB + (yc1 * EROW + 4 * w + t4) * 4));
            xres[0] = a0.x + c0.x; xres[1] = a0.y + c0.y; xres[2] = a1.x + c1.x; xres[3] = a1.y + c1.y;
            if (p.tanhEmbed) {
#pragma unroll
                for (int i = 0; i < 4; i++) xres[i] = wn::tanhf_fast(xres[i]);
            }
            const uint32_t x01 = pack_h2(xres[0], xres[1]), x23 = pack_h2(xres[2], xres[3]);
            sts64(sm + C::O_XBUF + xchg, x01, x23);
            stg_v2(gring + ring_off<WIDE>(it0.slot * L, rstride) + jw * 512 + hw * 8, x01, x23);
            // previous-index rows of the NEXT sample (= this sample's current index): global -> shared, asynchronously
            const unsigned char* ep = static_cast<const unsigned char*>(c.embPrev);
            const uint32_t en = sm + C::O_EPBUF + (epar ^ 1) * (TU * EROW * 4);
            cp_async4(en + (g * EROW + 4 * w + t4) * 4, ep + (size_t)yc0 * 128 + (4 * w + t4) * 4);
            cp_async4(en + ((g + 8) * EROW + 4 * w + t4) * 4, ep + (size_t)yc1 * 128 + (4 * w + t4) * 4);
            cp_async_commit();
        }
        bar_compute();
#pragma unroll
        for (int j = 0; j < 4; j++) load_a(xa[j], sm + C::O_XBUF + j * 512 + lane16);
        if (tid == 0) TRACE(0, 2);

        for (int l = 0; l < L; l++) step(t, l);
        ok_f1 = ok_f2 = false;                     // those looks were at slots the output pieces use first (same parity): stale

        // ---------------- relu(skip + bias) -> Zs -> Za   (reference.cpp:93-104)
#pragma unroll
        for (int i = 0; i < C::NSK; i++) {
            const int nt = w * C::NSK + i;
            uint32_t lo, hi;
            relu_skip(sk[i], s_bout, 8 * nt + 2 * t4, lo, hi);
            sts64(sm + C::O_OB0 + (nt >> 1) * 512 + lane16 + (nt & 1) * 8, lo, hi);
        }
        bar_compute();
        if (tid == 0) TRACE(0, 20);
        float zz[4][4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int c = 32 * w + 8 * i + 2 * t4;
            zz[i][0] = zz[i][2] = s_bout[S + c]; zz[i][1] = zz[i][3] = s_bout[S + c + 1];
        }
        // the 8 output pieces continue the ring sequence: piece q sits in slot type q & 1, slot sb ^ (q >> 1 & 1)
        auto out_gemm = [&](const int q, const int ojp, const uint32_t abuf, const int kp0) {
            const uint32_t idx = sb ^ ((q >> 1) & 1), bo = C::ring_bar(q & 1, idx);
            const uint32_t st = ((q & 1) ? sm + C::O_RING2 + idx * C::SLOT2 : sm + C::O_RING1 + idx * C::SLOT1) + o_out * ojp + lane16;
            mbar_wait(s_full + bo, fph ^ (((sb + (q >> 1)) >> 1) & 1));
            for (int jp = 0; jp < ojp; jp++) {
                uint32_t a0[4], a1[4];
                load_a(a0, abuf + ((kp0 + jp) * 2) * 512 + lane16);
                load_a(a1, abuf + ((kp0 + jp) * 2 + 1) * 512 + lane16);
                uint4 bw[4];
#pragma unroll
                for (int i = 0; i < 4; i++) bw[i] = lds128(st + (i * ojp + jp) * 512);
#pragma unroll
                for (int i = 0; i < 4; i++) hmma(zz[i], a0, bw[i].x, bw[i].y);
#pragma unroll
                for (int i = 0; i < 4; i++) hmma(zz[i], a1, bw[i].z, bw[i].w);
            }
            release(s_empty + bo);
        };
#pragma unroll
        for (int q = 0; q < C::NQ_ZS; q++) out_gemm(q, C::OJP_ZS, sm + C::O_OB0, q * C::OJP_ZS);
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int nt = 4 * w + i, c = 8 * nt + 2 * t4;
            const float z0 = fmaxf(zz[i][0], 0.f), z1 = fmaxf(zz[i][1], 0.f), z2 = fmaxf(zz[i][2], 0.f), z3 = fmaxf(zz[i][3], 0.f);
            sts64(sm + C::O_OB1 + (nt >> 1) * 512 + lane16 + (nt & 1) * 8, pack_h2(z0, z1), pack_h2(z2, z3));
            if (DUMP) {
                if (v0) { p.Zs[(size_t)b0 * A + c] = z0; p.Zs[(size_t)b0 * A + c + 1] = z1; }
                if (v1) { p.Zs[(size_t)b1 * A + c] = z2; p.Zs[(size_t)b1 * A + c + 1] = z3; }
            }
            zz[i][0] = zz[i][2] = s_bout[S + A + c]; zz[i][1] = zz[i][3] = s_bout[S + A + c + 1];
        }
        bar_compute();
        if (tid == 0) TRACE(0, 21);
#pragma unroll
        for (int q = 0; q < C::NQ_ZA; q++) out_gemm(C::NQ_ZS + q, C::OJP_ZA, sm + C::O_OB1, q * C::OJP_ZA);
        // 8 pieces = 4 slot pairs later: same slot, same barrier parity as before the output phase
        // logits (fp32) -> transposed buffer: row = utterance, 256 contiguous classes
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int c = 32 * w + 8 * i + 2 * t4;
            sts64(sm + C::O_LBUF + (g * LROW + c) * 4, __float_as_uint(zz[i][0]), __float_as_uint(zz[i][1]));
            sts64(sm + C::O_LBUF + ((g + 8) * LROW + c) * 4, __float_as_uint(zz[i][2]), __float_as_uint(zz[i][3]));
            if (DUMP) {
                if (v0) { p.Za[(size_t)b0 * A + c] = zz[i][0]; p.Za[(size_t)b0 * A + c + 1] = zz[i][1]; }
                if (v1) { p.Za[(size_t)b1 * A + c] = zz[i][2]; p.Za[(size_t)b1 * A + c + 1] = zz[i][3]; }
            }
        }
        bar_compute();
        if (tid == 0) TRACE(0, 22);
        if (t + 1 < t_end) {                       // every output piece is consumed: the first pieces of the next sample
            ok_f1 = probe(s_full + C::ring_bar(0, sb), fph);
            ok_f2 = probe(s_full + C::ring_bar(1, sb), fph);
        }
        // ---------------- softmax + categorical sample (matrix.cpp:167-183, reference.cpp:106-121): warp w serves
        // utterances 2w and 2w+1; lane holds 8 consecutive classes of each
        {
            // the max starts from the row's own logits, not at 0 as the CPU model's does (matrix.cpp:171): ex2.approx.ftz flushes
            // 2^(z - m) below 2^-126, so with a start at 0 a row whose logits all lie below about -87 would sum to 0
            float e[2][8], m[2];
#pragma unroll
            for (int r = 0; r < 2; r++) {
                const uint4 u0 = lds128(sm + C::O_LBUF + ((2 * w + r) * LROW + 8 * lane) * 4), u1 = lds128(sm + C::O_LBUF + ((2 * w + r) * LROW + 8 * lane + 4) * 4);
                e[r][0] = __uint_as_float(u0.x); e[r][1] = __uint_as_float(u0.y); e[r][2] = __uint_as_float(u0.z); e[r][3] = __uint_as_float(u0.w);
                e[r][4] = __uint_as_float(u1.x); e[r][5] = __uint_as_float(u1.y); e[r][6] = __uint_as_float(u1.z); e[r][7] = __uint_as_float(u1.w);
                m[r] = e[r][0];
#pragma unroll
                for (int k = 1; k < 8; k++) m[r] = fmaxf(m[r], e[r][k]);
            }
#pragma unroll
            for (int o = 16; o >= 1; o >>= 1) {
                m[0] = fmaxf(m[0], __shfl_xor_sync(0xffffffffu, m[0], o));
                m[1] = fmaxf(m[1], __shfl_xor_sync(0xffffffffu, m[1], o));
            }
            float incl[2];
#pragma unroll
            for (int r = 0; r < 2; r++) {
                const float ms = m[r] * 1.4426950408889634f;
                float run = 0.f;
#pragma unroll
                for (int k = 0; k < 8; k++) {
                    const float ev = wn::exp2f_fast(fmaf(e[r][k], 1.4426950408889634f, -ms));
                    run += ev;
                    e[r][k] = run;                                     // inclusive running sum inside the lane
                }
                incl[r] = run;
            }
            const float tot_lane[2] = {incl[0], incl[1]};
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const float a0 = __shfl_up_sync(0xffffffffu, incl[0], o), a1 = __shfl_up_sync(0xffffffffu, incl[1], o);
                if (lane >= o) { incl[0] += a0; incl[1] += a1; }
            }
#pragma unroll
            for (int r = 0; r < 2; r++) {
                const float total = __shfl_sync(0xffffffffu, incl[r], 31);
                const float excl = incl[r] - tot_lane[r];
                const float target = (r == 0 ? sel0 : sel1) * total;
                int cntk = 0;
#pragma unroll
                for (int k = 0; k < 8; k++) cntk += (target < excl + e[r][k]) ? 0 : 1;
                const unsigned ball = __ballot_sync(0xffffffffu, target < incl[r]);
                const int lf = ball ? __ffs(ball) - 1 : 31;
                const int ck = __shfl_sync(0xffffffffu, cntk, lf);
                const int y = ball ? 8 * lf + (ck < 7 ? ck : 7) : A - 1;
                const int b = tile * TU + 2 * w + r;
                if (DUMP && b < B) {
                    const float inv = 1.f / total;
                    float prevv = 0.f;
#pragma unroll
                    for (int k = 0; k < 8; k++) { p.P[(size_t)b * A + 8 * lane + k] = (e[r][k] - prevv) * inv; prevv = e[r][k]; }
                }
                if (lane == 0) {
                    int fbk = y;
                    if (b < B) {
                        p.yOut[(size_t)b * p.N + t] = y;
                        if (p.forced) fbk = p.forced[(size_t)b * p.N + t];
                    } else fbk = 128;
                    ys[TU + 2 * w + r] = ys[2 * w + r];
                    ys[2 * w + r] = fbk;
                }
            }
        }
        cp_async_wait_all();                       // the next sample's previous-index rows have landed
        bar_compute();
        if (tid == 0) TRACE(0, 23);
        epar ^= 1;
        if (++it0.slot == slots) it0.slot = 0;
        it0.t++;
    }
    store_ys(p, B, ys, tile * TU, tid);
}

// DUMP: write the last-sample activations (the host runs the final sample of a dumping launch with this variant).
// TRC:  record the clock64 timeline (debug; tools/lat_trace.py).
// MODELS: p.group_model is set, and the tile's weights are its group's model's (DESIGN.md §6).
// WIDE: the history ring passes 4 GiB, and its offsets are formed in 64 bits (ring_off).
template <int S, bool DUMP, bool TRC, bool MODELS, bool WIDE>
__global__ void __launch_bounds__(NT, 1) wn_lat_kernel(const WnParams p, const unsigned char* __restrict__ img0, const int ntiles_alloc)
{
    using C = Cfg<S>;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const uint32_t sm = smem_u32(smem_raw);
    const int L = p.L, B = p.B;
    const LatImage im = lat_image(S, L);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int tile = blockIdx.x;
    const WnGroupWeights gw = MODELS ? wn_group_weights(p, tile * TU) : WnGroupWeights{0, img0};
    const unsigned char* __restrict__ img = gw.image;
    const int slots = p.maxDil + 1;
    const int t_begin = p.init_sample, t_end = p.init_sample + p.count;
    const float* gbias = reinterpret_cast<const float*>(img + im.off_bias);
    const uint32_t s_full = sm + C::O_BAR + C::B_FULL, s_empty = sm + C::O_BAR + C::B_EMPTY, s_pfull = sm + C::O_BAR + C::B_PFULL;
    int* dil = reinterpret_cast<int*>(smem_raw + C::O_DIL);
    int* ys = reinterpret_cast<int*>(smem_raw + C::O_YS);
    float* s_bout = reinterpret_cast<float*>(smem_raw + C::O_BOUT);
    unsigned long long* trc = (TRC && p.trace && blockIdx.x == 0) ? p.trace : nullptr;
    int trn = 0;
    const int tr_t = p.trace_t & 0xFFFF;

    if (tid == 0) {
        for (int i = 0; i < C::NSLOT; i++) { mbar_init(s_full + 8 * i, 1); mbar_init(s_empty + 8 * i, NCW); }
        for (int i = 0; i < C::NPST; i++) mbar_init(s_pfull + 8 * i, 128);
        fence_mbar_init();
        int d = 1;                                     // dilation of layer l (nv_wavenet.cuh:99-111): 1,2,4..maxDil,1,2,...
        for (int l = 0; l < L; l++) { dil[l] = d; d <<= 1; if (d > p.maxDil) d = 1; }
    }
    {   // current-index embedding table -> shared memory (rows padded to 33 words: gathers of different rows fall into
        // different banks); output-layer biases; feedback state
        const uint32_t* ec = gw.at<uint32_t>(p.embCur);
        for (int i = tid; i < A * 32; i += NT) sts32(sm + C::O_EMB + ((i >> 5) * EROW + (i & 31)) * 4, ec[i]);
        for (int i = tid; i < S; i += NT) s_bout[i] = gbias[im.b_skpre + (size_t)(L - 1) * S + i];
        for (int i = tid; i < A; i += NT) { s_bout[S + i] = gbias[im.b_bzs + i]; s_bout[S + A + i] = gbias[im.b_bza + i]; }
        if (tid < TU) {
            const int b = tile * TU + tid;
            ys[tid] = b < B ? p.yCur[b] : 128;
            ys[TU + tid] = b < B ? p.yPrev[b] : 128;
        }
    }
    __syncthreads();

    const LatCta c{p, img, gw.at<void>(p.embPrev), im, sm, L, B, tid, warp, lane, tile, slots, t_begin, t_end, gbias, s_full, s_empty, s_pfull, dil, ys, s_bout, trc, tr_t};
    if (warp == NCW) {
        if (lane == 0) lat_producer<S, TRC>(c, trn);
    } else {
        lat_compute<S, DUMP, TRC, WIDE>(c, trn, ntiles_alloc);
    }
}
#undef TRACE

// ================================================================================================ three-CTA cluster variant
// The single-CTA kernel above runs at ~83 % of its SM's shared-memory bandwidth (per layer step: 72 KB written by TMA, 72 KB of
// B fragments and 48 KB of A fragments read back; ncu: 0.57 LSU wavefronts per cycle + the TMA writes).  Here one 16-utterance tile
// is served by a CLUSTER OF THREE CTAs on three SMs, and only what depends on the previous sample stays on the first one:
//   rank 0 "chain": embedding, cur / res GEMMs, gate, history ring writes             ring pieces [Wcur_l | Wres_l] (24 KB)
//   rank 1 "tail":  skip GEMM of every step (off the chain), output columns 0-127 of   ring pieces Wskip_l
//                   Zs and Za, softmax, sampling
//   rank 2 "prep":  (Bh + Lh) + Wprev . x[t-d] of the steps to come, up to NAP ahead;  ring pieces Wprev_l (16 KB)
//                   output columns 128-255 of Zs and Za, between two of its steps
// In the chain CTA a sync warp does every mbarrier wait and hand-back of the layer loop and enters the compute warps' named barriers
// behind what it saw land, so that a compute warp's layer step is its loads, HMMAs, gate, residual and the two barriers.
// The output weights stay resident: every compute thread of the tail and prep CTAs loads the B fragments of its two n-tiles once, at
// kernel start, Wzs into registers (S / 4) and Wza into its CTA's shared memory (64 KB per CTA).
// Distributed shared memory carries six flows, all as st.async with complete_tx on a transaction barrier that the receiver arms
// one phase ahead (data and signal travel together, no release fence on the sender), buffers handed back with relaxed remote arrives:
// h (2 KB per step, chain -> tail), the pre-activation before the current-sample GEMM (8 KB per step, prep -> chain), the 16 sampled
// indices (once per sample, tail -> chain); once per sample for the output layers: relu(skip + Bskip) (S x 32 B, tail -> prep),
// the relu(Zs) halves (4 KB each way, tail <-> prep) and the prep's logits half (8 KB fp32, prep -> tail).  Each CTA moves less than
// ~100 KB per step through its shared memory; a single CTA doing all of it moves ~190 KB per step and is bound by that.
// TR = utterances per cluster, 16 or 8.  An 8-row cluster c serves half c & 1 of 16-row tile c >> 1 of the conditioning store and the
// history ring (their layouts do not change: it reads and writes only its rows' words), keeps its shared-memory tiles at 8 rows and
// moves half the bytes of every flow above; the weights, and so the HMMAs and the B-fragment reads, are the same.
template <int S, int TR>
struct CfgC {
    using C = Cfg<S>;
    static_assert(TR == 16 || TR == 8, "a cluster serves 16 or 8 utterances");
    static constexpr uint32_t PIECE0 = 24576;                              // chain: [Wcur | Wres]
    // The chain's compute warps read the Wcur fragments of step n + 1 behind the h barrier of step n (8-row clusters), or those of
    // step n behind the x barrier of step n (16-row clusters, which measured 2 % slower reading them ahead: DESIGN §5.1b).
    static constexpr bool WCUR_AHEAD = TR == 8;
    // chain ring slots: piece n (step n) sits in slot n % NSLOT0.  Read ahead, piece n + 1 must have landed before the h barrier of
    // step n, and its slot is handed back behind the h barrier of step n + 1 - NSLOT0: the producer has NSLOT0 - 1 steps to refill
    // it.  With two slots (one step) the chain waits for the ring.
    static constexpr int NSLOT0 = WCUR_AHEAD ? 3 : 2;
    static_assert(NSLOT0 == 2 || NSLOT0 == 3, "the chain ring has two or three slots");
    __device__ static __forceinline__ uint32_t slot0(uint32_t n) { return n % NSLOT0; }
    __device__ static __forceinline__ uint32_t par0(uint32_t n) { return (n / NSLOT0) & 1; }   // phase parity of piece n's fill
    static constexpr uint32_t SLOT1 = S * 128;                             // tail: Wskip_l
    static constexpr int NSLOT1 = 3;
    static constexpr int NAP = 4;                                          // pre-activation tiles in flight from the prep CTA to the chain CTA
    static constexpr int NPS = 8;                                          // staged history / conditioning tiles of the prep CTA
    static constexpr int NPRING = 4;                                       // Wprev ring slots of the prep CTA
    static constexpr int NHB = 2;                                          // h tiles in flight from the chain CTA to the tail CTA
    static constexpr int NRING = NSLOT1 > NPRING ? NSLOT1 : NPRING;        // weight-ring barrier pairs (the chain uses NSLOT0)
    static_assert(NSLOT0 <= NRING, "the chain ring's barriers fit the reserved pairs");
    static_assert((NAP & (NAP - 1)) == 0 && (NPS & (NPS - 1)) == 0 && (NPRING & (NPRING - 1)) == 0 && (NHB & (NHB - 1)) == 0,
                  "slot counts are powers of two, so that slot and parity arithmetic stays a mask and a shift");
    static constexpr int RPW = TR / NCW;                                   // rows sampled per tail warp
    static constexpr uint32_t XT = TR * 128;                               // activation tile (x, h, x[t-d]): TR rows x 64 channels fp16
    static constexpr uint32_t AP = TR * 512;                               // pre-activation tile: TR rows x 128 channels fp32
    // chain CTA
    static constexpr uint32_t C_RING = 0;                                  // NSLOT0 x PIECE0
    static constexpr uint32_t C_EMB = NSLOT0 * PIECE0;
    static constexpr uint32_t C_EPBUF = C_EMB + A * EROW * 4;
    static constexpr uint32_t C_XBUF = C_EPBUF + 2 * TR * EROW * 4;
    static constexpr uint32_t C_HBUF = C_XBUF + XT;
    static constexpr uint32_t C_AP = C_HBUF + XT;                          // NAP x AP: (Bh + Lh) + Wprev . x[t-d] of the coming steps, written by the prep CTA
    static constexpr uint32_t C_BIAS = C_AP + NAP * AP;                    // [L][8 warps][4][8] fp32: Bh / Bres pairs per thread (Bres is read here)
    static constexpr uint32_t C_END = C_BIAS + MAXL * 1024;
    // tail CTA
    // Output layers, tail and prep CTAs: OB0 = relu(skip + Bskip) and OB1 = relu(Zs) in A-fragment order (OB1 k-steps 0-7 come from
    // the tail, 8-15 from the prep; each CTA writes into the other's), ZA = this CTA's half of Wza in B-fragment order, resident.
    static constexpr uint32_t OB0_BYTES = (S / 16) * 32 * TR, OB1_BYTES = (A / 16) * 32 * TR, ZA_BYTES = 16 * (A / 32) * 512;
    static constexpr uint32_t T_RING = 0;                                  // NSLOT1 x SLOT1
    static constexpr uint32_t T_HBUF = NSLOT1 * SLOT1;                     // NHB x XT, written by the chain CTA
    static constexpr uint32_t T_LBUF = T_HBUF + NHB * XT;                    // transposed logits; columns 128-255 written by the prep CTA
    static constexpr uint32_t T_BOUT = T_LBUF + TR * LROW * 4;             // fp32: Bskip total [S], Bzs [A], Bza [A]
    static constexpr uint32_t T_OB0 = T_BOUT + (S + 2 * A) * 4;
    static constexpr uint32_t T_OB1 = T_OB0 + OB0_BYTES;
    static constexpr uint32_t T_ZA = T_OB1 + OB1_BYTES;
    static constexpr uint32_t T_END = T_ZA + ZA_BYTES;
    // prep CTA
    static constexpr uint32_t P_RING = 0;                                  // NPRING x 16 KB: Wprev_l
    // (both staged as whole 16-row tiles at either height: see the prep CTA's staging)
    static constexpr uint32_t P_PST = NPRING * 16384;                      // NPS x 2 KB: staged history tiles x[t-d] (A-fragment order)
    static constexpr uint32_t P_COND = P_PST + NPS * 2048;                 // NPS x 4 KB: conditioning tiles, staged with the history tiles (cp.async)
    static constexpr uint32_t P_BIAS = P_COND + NPS * 4096;                // [L][8 warps][4][4] fp32: this thread's Bh
    static constexpr uint32_t P_DIL = P_BIAS + MAXL * 512;
    static constexpr uint32_t P_BOUT = P_DIL + MAXL * 4;                   // fp32: Bzs [A], Bza [A]
    static constexpr uint32_t P_OB0 = P_BOUT + 2 * A * 4;
    static constexpr uint32_t P_OB1 = P_OB0 + OB0_BYTES;
    static constexpr uint32_t P_ZA = P_OB1 + OB1_BYTES;
    static constexpr uint32_t P_END = P_ZA + ZA_BYTES;
    // common tail of the maps (same offsets in every CTA, so that remote addresses are computed with mapa on local ones)
    static_assert(C_END <= P_END, "the chain's map (its ring included) stays below the prep CTA's, so the ring depth does not grow SMEM");
    static constexpr uint32_t O_YS = (C_END > T_END ? (C_END > P_END ? C_END : P_END) : (T_END > P_END ? T_END : P_END));
    static constexpr uint32_t O_BAR = O_YS + 2 * TR * 4;
    static constexpr uint32_t SMEM = O_BAR + 40 * 8;
    static_assert(SMEM <= 227 * 1024, "the cluster kernel's shared-memory map exceeds the 227 KB an H100 CTA may use");
    // mbarriers at O_BAR (what each one guards: wn_lat2_kernel)
    static constexpr uint32_t B_FULL = 0, B_EMPTY = B_FULL + NRING * 8, B_PFULL = B_EMPTY + NRING * 8;
    static constexpr uint32_t B_HFULL = B_PFULL + NPS * 8, B_HFREE = B_HFULL + NHB * 8, B_YFULL = B_HFREE + NHB * 8;
    static constexpr uint32_t B_APFULL = B_YFULL + 8, B_APFREE = B_APFULL + NAP * 8;
    static constexpr uint32_t B_OB0FULL = B_APFREE + NAP * 8, B_OB0FREE = B_OB0FULL + 8, B_OB1FULL = B_OB0FREE + 8, B_OB1FREE = B_OB1FULL + 8;
    static constexpr uint32_t B_LFULL = B_OB1FREE + 8, B_LFREE = B_LFULL + 8, B_END = B_LFREE + 8;
    static_assert(O_BAR + B_END <= SMEM, "the mbarriers outgrow their reservation");
};
constexpr int NCL = 3;                       // CTAs per cluster
constexpr int NTC = NT + 32;                 // threads of a cluster CTA: + the chain CTA's sync warp (idle in the tail and prep CTAs)

__device__ __forceinline__ uint32_t mapa_u32(uint32_t addr, uint32_t rank)
{
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
    return r;
}
// remote stores that complete bytes on a remote mbarrier (data and signal travel together: no release fence on the sender)
__device__ __forceinline__ void st_async_b32(uint32_t raddr, uint32_t a, uint32_t rbar)
{
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(raddr), "r"(a), "r"(rbar) : "memory");
}
__device__ __forceinline__ void st_async_v2(uint32_t raddr, uint32_t a, uint32_t b, uint32_t rbar)
{
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v2.b32 [%0], {%1,%2}, [%3];" ::"r"(raddr), "r"(a), "r"(b), "r"(rbar) : "memory");
}
__device__ __forceinline__ void st_async_v4(uint32_t raddr, uint4 v, uint32_t rbar)
{
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1,%2,%3,%4}, [%5];"
                 ::"r"(raddr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "r"(rbar) : "memory");
}
__device__ __forceinline__ void st_async_v4(uint32_t raddr, float a, float b, float c, float d, uint32_t rbar)
{
    st_async_v4(raddr, make_uint4(__float_as_uint(a), __float_as_uint(b), __float_as_uint(c), __float_as_uint(d)), rbar);
}
// "this buffer is free again": no data behind it, so no release ordering is paid for
__device__ __forceinline__ void mbar_arrive_remote(uint32_t raddr) { asm volatile("mbarrier.arrive.relaxed.cluster.shared::cluster.b64 _, [%0];" ::"r"(raddr) : "memory"); }
__device__ __forceinline__ void cluster_sync_all()
{
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// the warp is done with a buffer: one arrival (lane 0, after the warp's reads) on its barrier here / in cluster CTA `rank`
__device__ __forceinline__ void release(uint32_t bar, int lane) { __syncwarp(); if (lane == 0) mbar_arrive(bar); }
__device__ __forceinline__ void release_remote(uint32_t local_bar, uint32_t rank, int lane)
{
    __syncwarp();
    if (lane == 0) mbar_arrive_remote(mapa_u32(local_bar, rank));
}

// What more than one role of wn_lat2_kernel uses; set once, by the kernel's prologue.
struct ClusterCta {
    const WnParams& p;
    const unsigned char* img;                   // the cluster's weight image and previous-index embedding table (its model's)
    const void* embPrev;
    LatImage im;
    unsigned char* smem;                        // shared memory, and its shared-window address
    uint32_t sm;
    int L, B, tid;
    uint32_t crank;                             // cluster rank: 0 chain, 1 tail, 2 prep
    int ub, tile;                               // utterances ub .. ub + TR - 1, in 16-row tile `tile` (hw4: see the kernel)
    uint32_t hw4;
    int slots, t_begin, t_end, ntiles_alloc;
    const float* gbias;
    uint32_t s_full, s_empty, s_pfull, s_hfull, s_hfree, s_yfull, s_apfull, s_apfree;      // mbarriers: CfgC::B_*
    uint32_t s_ob0full, s_ob0free, s_ob1full, s_ob1free, s_lfull, s_lfree;
    int* ys;                                    // [TR] current index, [TR] previous index
    // this thread: warp w, lane = 4 g + t4, rows b0 and b1 (v0, v1: inside the batch), lane16 = 16 lane, its slot of an activation tile
    int w, lane, g, t4, b0, b1;
    bool v0, v1;
    uint32_t lane16, xchg;
    unsigned long long* trc;                    // debug timeline: see the kernel
    int tr_t;
};
#define TRACE2(role, tag) do { if (TRC && trc && threadIdx.x == 0 && t == tr_t && trn < 1023) trc[(role) * 1024 + trn++] = ((unsigned long long)(tag) << 48) | (clock64() & 0xFFFFFFFFFFFFull); } while (0)

// ---------------- output layers, tail (half 0) and prep (half 1) CTAs: n-tiles 16 half + 2w and 16 half + 2w + 1 of Zs and Za.
// Their B fragments (lat_pack_kernel: piece q of a matrix = k-step pairs [q OJP, (q+1) OJP) of all 32 n-tiles, fragment
// (n-tile OJP + jp) x 512 + lane x 16) are loaded once, at kernel start: Wzs into registers (S / 4 per thread), Wza into this
// CTA's ZA region, where every thread reads back only the 16 B it stored itself (fragment (2w + i) x A/32 + jp).  Wza resident
// in registers as well would not fit: ten warps leave 168 registers per thread (three warps share a sub-partition's 64 KB),
// and the tail's skip loop and the prep's step loop would spill ~300 B at S = 256.
template <int S, int TR>
__device__ __forceinline__ void load_out_w(const ClusterCta& c, uint4 (&zsw)[2][S / 32], const uint32_t half)
{
    using C = Cfg<S>;
    using M = CfgC<S, TR>;
    const unsigned char* img = c.img;
    const LatImage& im = c.im;
    const uint32_t sm = c.sm, lane16 = c.lane16;
    const int w = c.w;
    const uint32_t za = sm + (half ? M::P_ZA : M::T_ZA) + lane16;
#pragma unroll
    for (int i = 0; i < 2; i++) {
        const int nt = 16 * half + 2 * w + i;
#pragma unroll
        for (int jp = 0; jp < S / 32; jp++)
            zsw[i][jp] = ldg_nc_v4(img + im.off_zs + (size_t)(jp / C::OJP_ZS) * C::ZS_PIECE + (size_t)(nt * C::OJP_ZS + jp % C::OJP_ZS) * 512 + lane16);
        for (int jp = 0; jp < A / 32; jp++)
            sts128(za + ((2 * w + i) * (A / 32) + jp) * 512,
                   ldg_nc_v4(img + im.off_za + (size_t)(jp / C::OJP_ZA) * C::ZA_PIECE + (size_t)(nt * C::OJP_ZA + jp % C::OJP_ZA) * 512 + lane16));
    }
}
// relu(skip + Bskip) is in this CTA's OB0 (the prep waits for it here).  Per n-tile the HMMAs run from the bias through the
// k-steps in order on one accumulator, as in the single-CTA kernel.  relu(Zs) of the two n-tiles is k-step 8 half + w of the
// Za GEMM's A operand: 16 B per thread into this CTA's OB1 and the peer's.  Leaves the logits of the two n-tiles in zz.
template <int S, int TR, bool DUMP, bool TRC>
__device__ __forceinline__ void out_half(const ClusterCta& c, int& trn, const int t, const uint4 (&zsw)[2][S / 32], const uint32_t half, float (&zz)[2][4])
{
    using M = CfgC<S, TR>;
    const WnParams& p = c.p;
    unsigned char* smem_raw = c.smem;
    const uint32_t sm = c.sm, crank = c.crank, lane16 = c.lane16;
    const uint32_t s_ob0full = c.s_ob0full, s_ob0free = c.s_ob0free, s_ob1full = c.s_ob1full, s_ob1free = c.s_ob1free;
    const int tid = c.tid, t_begin = c.t_begin, w = c.w, lane = c.lane, t4 = c.t4, b0 = c.b0, b1 = c.b1;
    const bool v0 = c.v0, v1 = c.v1;
    unsigned long long* trc = c.trc;
    const int tr_t = c.tr_t;
    const uint32_t peer = half ? 1 : 2, par = (uint32_t)(t - t_begin) & 1;
    const float* bz = reinterpret_cast<const float*>(smem_raw + (half ? M::P_BOUT : M::T_BOUT + S * 4));   // Bzs [A], Bza [A]
    const uint32_t ob0 = sm + (half ? M::P_OB0 : M::T_OB0), ob1 = sm + (half ? M::P_OB1 : M::T_OB1), za = sm + (half ? M::P_ZA : M::T_ZA);
#pragma unroll
    for (int i = 0; i < 2; i++) {
        const int c = 8 * (16 * (int)half + 2 * w + i) + 2 * t4;
        zz[i][0] = zz[i][2] = bz[c]; zz[i][1] = zz[i][3] = bz[c + 1];
    }
    // the Wza fragments of the first half of K (32 registers) are read while the CTA would wait anyway: the prep before relu(skip)
    // arrives, the tail after its Zs HMMAs, while the prep's relu(Zs) half is still on its way; those of the second half inside
    // the Za GEMM (three quarters or more up front spill at S = 256)
    constexpr int ZPRE = A / 64;
    uint4 zab[2][A / 32];
    auto load_za = [&]() {
#pragma unroll
        for (int jp = 0; jp < ZPRE; jp++)
#pragma unroll
            for (int i = 0; i < 2; i++) zab[i][jp] = lds128(za + ((2 * w + i) * (A / 32) + jp) * 512 + lane16);
    };
    if (half) { load_za(); mbar_wait(s_ob0full, par); }
#pragma unroll
    for (int jp = 0; jp < S / 32; jp++) {
        uint32_t a0[4], a1[4];
        load_a_rows<TR>(a0, ob0, 2 * jp, lane);
        load_a_rows<TR>(a1, ob0, 2 * jp + 1, lane);
#pragma unroll
        for (int i = 0; i < 2; i++) hmma(zz[i], a0, zsw[i][jp].x, zsw[i][jp].y);
#pragma unroll
        for (int i = 0; i < 2; i++) hmma(zz[i], a1, zsw[i][jp].z, zsw[i][jp].w);
    }
    if (!half) load_za();
    if (half) {                                    // OB0 has been read: arm its barrier for the next sample, then free it
        if (tid == 0) mbar_arrive_expect_tx(s_ob0full, TR * S * 2);
        release_remote(s_ob0free, 1, lane);
    }
    TRACE2(crank, 24);
    uint32_t zp[4];
#pragma unroll
    for (int i = 0; i < 2; i++) {
        const int c = 8 * (16 * (int)half + 2 * w + i) + 2 * t4;
        const float z0 = fmaxf(zz[i][0], 0.f), z1 = fmaxf(zz[i][1], 0.f), z2 = fmaxf(zz[i][2], 0.f), z3 = fmaxf(zz[i][3], 0.f);
        zp[2 * i] = pack_h2(z0, z1); zp[2 * i + 1] = pack_h2(z2, z3);
        if (DUMP) {
            if (v0) { p.Zs[(size_t)b0 * A + c] = z0; p.Zs[(size_t)b0 * A + c + 1] = z1; }
            if (v1) { p.Zs[(size_t)b1 * A + c] = z2; p.Zs[(size_t)b1 * A + c + 1] = z3; }
        }
        zz[i][0] = zz[i][2] = bz[A + c]; zz[i][1] = zz[i][3] = bz[A + c + 1];
    }
    {   // both CTAs' warps have read the previous sample's OB1
        const uint32_t o = (uint32_t)((8 * half + w) * 32 * TR + lane * TR);      // k-step 8 half + w of OB1
        const uint32_t ro = mapa_u32(sm + (half ? M::T_OB1 : M::P_OB1) + o, peer), rbar = mapa_u32(s_ob1full, peer);
        mbar_wait(s_ob1free, par ^ 1);
        if (TR == TU) {
            const uint4 v = make_uint4(zp[0], zp[1], zp[2], zp[3]);
            sts128(ob1 + o, v);
            st_async_v4(ro, v, rbar);
        } else {
            sts64(ob1 + o, zp[0], zp[2]);
            st_async_v2(ro, zp[0], zp[2], rbar);
        }
    }
    bar_compute();
    mbar_wait(s_ob1full, par);
    TRACE2(crank, 21);
#pragma unroll
    for (int jp = 0; jp < A / 32; jp++) {
        uint32_t a0[4], a1[4];
        load_a_rows<TR>(a0, ob1, 2 * jp, lane);
        load_a_rows<TR>(a1, ob1, 2 * jp + 1, lane);
        if (jp >= ZPRE) {
#pragma unroll
            for (int i = 0; i < 2; i++) zab[i][jp] = lds128(za + ((2 * w + i) * (A / 32) + jp) * 512 + lane16);
        }
#pragma unroll
        for (int i = 0; i < 2; i++) hmma(zz[i], a0, zab[i][jp].x, zab[i][jp].y);
#pragma unroll
        for (int i = 0; i < 2; i++) hmma(zz[i], a1, zab[i][jp].z, zab[i][jp].w);
    }
    // OB1 has been read: arm its barrier for the peer's next half, then free it for both CTAs
    if (tid == 0) mbar_arrive_expect_tx(s_ob1full, TR * 128 * 2);
    release(s_ob1free, lane);
    release_remote(s_ob1free, peer, lane);
    if (DUMP) {
#pragma unroll
        for (int i = 0; i < 2; i++) {
            const int c = 8 * (16 * (int)half + 2 * w + i) + 2 * t4;
            if (v0) { p.Za[(size_t)b0 * A + c] = zz[i][0]; p.Za[(size_t)b0 * A + c + 1] = zz[i][1]; }
            if (v1) { p.Za[(size_t)b1 * A + c] = zz[i][2]; p.Za[(size_t)b1 * A + c + 1] = zz[i][3]; }
        }
    }
}

// ===================================================================================== chain CTA
template <int S, int TR, bool DUMP, bool TRC, bool WIDE>
__device__ __forceinline__ void chain_cta(const ClusterCta& c, int& trn)
{
    using C = Cfg<S>;
    using M = CfgC<S, TR>;
    const WnParams& p = c.p;
    const unsigned char* img = c.img;
    const LatImage& im = c.im;
    const uint32_t sm = c.sm, hw4 = c.hw4, lane16 = c.lane16, xchg = c.xchg;
    const uint32_t s_full = c.s_full, s_empty = c.s_empty, s_hfull = c.s_hfull, s_hfree = c.s_hfree, s_yfull = c.s_yfull;
    const uint32_t s_apfull = c.s_apfull, s_apfree = c.s_apfree;
    const int L = c.L, B = c.B, tid = c.tid, tile = c.tile, slots = c.slots, t_begin = c.t_begin, t_end = c.t_end, ntiles_alloc = c.ntiles_alloc;
    const int w = c.w, lane = c.lane, g = c.g, t4 = c.t4, b0 = c.b0, b1 = c.b1;
    const int* ys = c.ys;
    unsigned long long* trc = c.trc;
    const int tr_t = c.tr_t;
    if (w == NCW) {
        if (lane == 0) {
            uint32_t pc = 0;
            for (int t = t_begin; t < t_end; t++)
                for (int l = 0; l < L; l++, pc++) {
                    const uint32_t sl = M::slot0(pc);
                    mbar_wait(s_empty + 8 * sl, M::par0(pc) ^ 1);
                    mbar_arrive_expect_tx(s_full + 8 * sl, M::PIECE0);
                    tma_load_1d(sm + M::C_RING + sl * M::PIECE0, img + (size_t)l * im.layer_bytes + C::W_CUR, 16384, s_full + 8 * sl);
                    tma_load_1d(sm + M::C_RING + sl * M::PIECE0 + 16384, img + (size_t)l * im.layer_bytes + C::W_RES, 8192, s_full + 8 * sl);
                }
        }
    } else if (w == NCW + 1) {
        // Sync warp: every mbarrier of the layer loop, so that the compute warps pass only their two named barriers per step.  Its
        // lane 0 enters a barrier once what the compute warps will read behind it has landed, and answers for what they have read
        // before it:
        //   before the first barrier: pre-activation tile 0 is full (WCUR_AHEAD: and ring piece 0);
        //   before the x barrier of step n: the tail's h buffer n % NHB is free (it has read tile n - NHB), so that every compute
        //     thread sends its words of h tile n with st.async behind that barrier (!WCUR_AHEAD: and ring piece n is full);
        //   after it: pre-activation tile n has been read (behind the h barrier of step n - 1): re-armed, handed back to the prep CTA;
        //   before the h barrier of step n: pre-activation tile n + 1 is full (WCUR_AHEAD: and ring piece n + 1); the compute warps
        //     read the tile (and piece n + 1's Wcur fragments) behind that barrier;
        //   after it: ring piece n has been read (its Wcur behind the h barrier of step n - 1 or the x barrier of step n, its Wres
        //     before this one): empty.
        const int nsteps = (t_end - t_begin) * L;
        const uint32_t r_apfree = mapa_u32(s_apfree, 2);
        if (lane == 0 && nsteps > 0) {
            mbar_wait(s_apfull, 0);
            if (M::WCUR_AHEAD) mbar_wait(s_full, 0);
        }
        bar_chain();
        for (int n = 0; n < nsteps; n++) {
            const uint32_t b = (uint32_t)n % M::NAP, hb = (uint32_t)n % M::NHB;
            if (lane == 0) {
                if (!M::WCUR_AHEAD) mbar_wait(s_full + 8 * M::slot0(n), M::par0(n));
                mbar_wait(s_hfree + 8 * hb, (((uint32_t)n / M::NHB) & 1) ^ 1);
            }
            __syncwarp();
            bar_chain();                                   // x barrier of step n
            if (lane == 0) {
                mbar_arrive_expect_tx(s_apfull + 8 * b, M::AP);    // armed for the tile NAP steps on, before the buffer goes back
                mbar_arrive_remote(r_apfree + 8 * b);
                if (n + 1 < nsteps) {
                    mbar_wait(s_apfull + 8 * ((uint32_t)(n + 1) % M::NAP), ((uint32_t)(n + 1) / M::NAP) & 1);
                    if (M::WCUR_AHEAD) mbar_wait(s_full + 8 * M::slot0(n + 1), M::par0(n + 1));
                }
            }
            __syncwarp();
            bar_chain();                                   // h barrier of step n
            if (lane == 0) mbar_arrive(s_empty + 8 * M::slot0(n));
        }
    } else if (w < NCW) {
        const uint32_t rstride = (uint32_t)ntiles_alloc * 2048u;
        unsigned char* gring = static_cast<unsigned char*>(p.ring) + (size_t)tile * 2048 + hw4;
        const int cw = 8 * w + 2 * t4;
        const int nsteps = (t_end - t_begin) * L;
        const uint32_t o_t0 = (uint32_t)(w * 2) * 512 + lane16, o_g0 = (uint32_t)((8 + w) * 2) * 512 + lane16, o_res = 16384u + (uint32_t)(w * 2) * 512 + lane16;
        const uint32_t r_hbuf = mapa_u32(sm + M::T_HBUF + xchg, 1);            // this thread's slot of the tail CTA's h tiles
        const uint32_t r_hfull = mapa_u32(s_hfull, 1);
        const uint32_t s_bias = sm + M::C_BIAS + (uint32_t)(w * 4 + t4) * 32;   // this thread's Bh / Bres pairs of layer 0 (+ 1 KB per layer)
        const uint32_t s_ap = sm + M::C_AP + (uint32_t)tid * (2 * TR);         // this thread's 2 TR / 4 floats of a pre-activation tile (+ AP per buffer)
        uint32_t xa[4][4];
        float accp[2][4];
        float2 brn = make_float2(0.f, 0.f);
        float xres[4] = {0.f, 0.f, 0.f, 0.f};
        // accp <- (Bh + Lh) + Wprev . x[t-d] of step n (layer l), computed by the prep CTA; brn <- Bres of layer l
        auto load_ap = [&](const uint32_t n, const int l) {
            const uint2 b2 = lds64(s_bias + l * 1024 + 16);
            const uint4 a0 = lds128(s_ap + (n % M::NAP) * M::AP);
            brn = make_float2(__uint_as_float(b2.x), __uint_as_float(b2.y));
            if (TR == TU) {
                const uint4 a1 = lds128(s_ap + (n % M::NAP) * M::AP + 16);
                accp[0][0] = __uint_as_float(a0.x); accp[0][1] = __uint_as_float(a0.y); accp[0][2] = __uint_as_float(a0.z); accp[0][3] = __uint_as_float(a0.w);
                accp[1][0] = __uint_as_float(a1.x); accp[1][1] = __uint_as_float(a1.y); accp[1][2] = __uint_as_float(a1.z); accp[1][3] = __uint_as_float(a1.w);
            } else {                                       // row g only: tanh pair, sigmoid pair
                accp[0][0] = __uint_as_float(a0.x); accp[0][1] = __uint_as_float(a0.y); accp[1][0] = __uint_as_float(a0.z); accp[1][1] = __uint_as_float(a0.w);
                accp[0][2] = accp[0][3] = accp[1][2] = accp[1][3] = 0.f;
            }
        };
        {   // prologue: previous-index rows of the first sample
            const uint32_t* ep = static_cast<const uint32_t*>(c.embPrev);
            sts32(sm + M::C_EPBUF + (g * EROW + 4 * w + t4) * 4, ep[ys[TR + g] * 32 + 4 * w + t4]);
            if (TR == TU) sts32(sm + M::C_EPBUF + ((g + 8) * EROW + 4 * w + t4) * 4, ep[ys[TU + g + 8] * 32 + 4 * w + t4]);
        }
        StepIt it0{t_begin, 0, p.ring_slot};
        bar_chain();                                       // pre-activation tile 0 (and ring piece 0) have landed
        // wc (WCUR_AHEAD): the Wcur fragments of the next step, read behind the h barrier of the step before (they are in a ring
        // piece the sync warp saw land), so that after the x barrier only the x tile is read before the cur HMMAs
        GateW wc{};
        if (nsteps > 0) {
            load_ap(0, 0);
            if (M::WCUR_AHEAD) wc = lds_gate_w(sm + M::C_RING, o_t0, o_g0);
        }
        auto load_wcur = [&](const uint32_t n1) {
            if (n1 < (uint32_t)nsteps) wc = lds_gate_w(sm + M::C_RING + M::slot0(n1) * M::PIECE0, o_t0, o_g0);
        };

        uint32_t n = 0, epar = 0;                          // step, sample parity
        for (int t = t_begin; t < t_end; t++) {
            TRACE2(0, 1);
            if (t > t_begin) {                             // the tail CTA has written this sample's indices into ys
                mbar_wait(s_yfull, (uint32_t)(t - t_begin - 1) & 1);
                if (tid == 0 && t + 1 < t_end) mbar_arrive_expect_tx(s_yfull, 2 * TR * 4);          // arm the next hand-back
            }
            {   // embedding (reference.cpp:42-57), this warp's 8 channels
                const int yc0 = ys[g], yc1 = TR == TU ? ys[g + 8] : 0;
                const uint32_t eo = sm + M::C_EPBUF + epar * (TR * EROW * 4);
                const unsigned char* ep = static_cast<const unsigned char*>(c.embPrev);
                const uint32_t en = sm + M::C_EPBUF + (epar ^ 1) * (TR * EROW * 4);
                const float2 a0 = unpack_h2(lds32(eo + (g * EROW + 4 * w + t4) * 4));
                const float2 c0 = unpack_h2(lds32(sm + M::C_EMB + (yc0 * EROW + 4 * w + t4) * 4));
                xres[0] = a0.x + c0.x; xres[1] = a0.y + c0.y;
                if (TR == TU) {
                    const float2 a1 = unpack_h2(lds32(eo + ((g + 8) * EROW + 4 * w + t4) * 4));
                    const float2 c1 = unpack_h2(lds32(sm + M::C_EMB + (yc1 * EROW + 4 * w + t4) * 4));
                    xres[2] = a1.x + c1.x; xres[3] = a1.y + c1.y;
                }
                if (p.tanhEmbed) {
#pragma unroll
                    for (int i = 0; i < (TR == TU ? 4 : 2); i++) xres[i] = wn::tanhf_fast(xres[i]);
                }
                store_x<TR, WIDE>(xres, sm + M::C_XBUF + xchg, gring + lane16, (uint32_t)(it0.slot * L), rstride, w);
                cp_async4(en + (g * EROW + 4 * w + t4) * 4, ep + (size_t)yc0 * 128 + (4 * w + t4) * 4);
                if (TR == TU) cp_async4(en + ((g + 8) * EROW + 4 * w + t4) * 4, ep + (size_t)yc1 * 128 + (4 * w + t4) * 4);
                cp_async_commit();                         // landed long before the next sample starts (waited for at the end of this one)
            }
            bar_chain();
#pragma unroll
            for (int j = 0; j < 4; j++) load_a_rows<TR>(xa[j], sm + M::C_XBUF, j, lane);
            TRACE2(0, 2);

            for (int l = 0; l < L; l++, n++) {
                const uint32_t p1 = sm + M::C_RING + M::slot0(n) * M::PIECE0;
                const float2 br = brn;
                {
                    if (!M::WCUR_AHEAD) wc = lds_gate_w(p1, o_t0, o_g0);
                    const uint4 bt0 = wc.t0, bg0 = wc.g0, bt1 = wc.t1, bg1 = wc.g1;
                    float u0[4] = {0.f, 0.f, 0.f, 0.f}, u1[4] = {0.f, 0.f, 0.f, 0.f};
                    hmma(accp[0], xa[0], bt0.x, bt0.y); hmma(accp[1], xa[0], bg0.x, bg0.y); hmma(u0, xa[2], bt1.x, bt1.y); hmma(u1, xa[2], bg1.x, bg1.y);
                    hmma(accp[0], xa[1], bt0.z, bt0.w); hmma(accp[1], xa[1], bg0.z, bg0.w); hmma(u0, xa[3], bt1.z, bt1.w); hmma(u1, xa[3], bg1.z, bg1.w);
#pragma unroll
                    for (int i = 0; i < 4; i++) { accp[0][i] += u0[i]; accp[1][i] += u1[i]; }
                }
                // the res GEMM's B fragments (same ring piece), read while the shared-memory pipe is idle under the HMMAs and the
                // gate, so that only the h tile is read between the barrier below and the res HMMAs
                const uint4 bw0 = lds128(p1 + o_res), bw1 = lds128(p1 + o_res + 512);
                {
                    uint32_t h01, h23;
                    gate<TR>(accp, sm + M::C_HBUF + xchg, h01, h23);
                    // the tail CTA's copy: buffer n % NHB, free since the x barrier (the sync warp)
                    if (TR == TU) st_async_v2(r_hbuf + (n % M::NHB) * M::XT, h01, h23, r_hfull + 8 * (n % M::NHB));
                    else st_async_b32(r_hbuf + (n % M::NHB) * M::XT, h01, r_hfull + 8 * (n % M::NHB));
                }
                TRACE2(0, 12);
                bar_chain();
                uint32_t ha[4][4];
#pragma unroll
                for (int j = 0; j < 4; j++) load_a_rows<TR>(ha[j], sm + M::C_HBUF, j, lane);
                TRACE2(0, 10);
                if (n + 1 < (uint32_t)nsteps) load_ap(n + 1, l + 1 < L ? l + 1 : 0);
                float ra[4] = {0.f, 0.f, 0.f, 0.f}, rb[4] = {0.f, 0.f, 0.f, 0.f};
                hmma_res(ra, rb, ha, bw0, bw1);
                residual<TR, WIDE>(xres, ra, rb, br, l + 1 < L, sm + M::C_XBUF + xchg, gring + lane16, (uint32_t)(it0.slot * L + l + 1), rstride, w);
                // after the x store, which the x barrier waits for, so that the store is not queued behind these loads (placed right
                // after the res HMMAs, the layer step measured slower: DESIGN §5.1b)
                if (M::WCUR_AHEAD) load_wcur(n + 1);
                TRACE2(0, 14);
                dump_xt<DUMP>(p, B, l, b0, b1, cw, xres);
                if (l + 1 < L) {
                    bar_chain();
#pragma unroll
                    for (int j = 0; j < 4; j++) load_a_rows<TR>(xa[j], sm + M::C_XBUF, j, lane);
                }
                TRACE2(0, 11);
            }
            cp_async_wait_all();                           // the previous-index rows of the next sample
            epar ^= 1;
            if (++it0.slot == slots) it0.slot = 0;
            it0.t++;
        }
    }
}

// ===================================================================================== tail CTA
template <int S, int TR, bool DUMP, bool TRC>
__device__ __forceinline__ void tail_cta(const ClusterCta& c, int& trn)
{
    using C = Cfg<S>;
    using M = CfgC<S, TR>;
    const WnParams& p = c.p;
    const unsigned char* img = c.img;
    const LatImage& im = c.im;
    unsigned char* smem_raw = c.smem;
    const uint32_t sm = c.sm, lane16 = c.lane16;
    const uint32_t s_full = c.s_full, s_empty = c.s_empty, s_hfull = c.s_hfull, s_hfree = c.s_hfree, s_yfull = c.s_yfull;
    const uint32_t s_ob0full = c.s_ob0full, s_ob0free = c.s_ob0free, s_lfull = c.s_lfull, s_lfree = c.s_lfree;
    const int L = c.L, B = c.B, tid = c.tid, ub = c.ub, t_begin = c.t_begin, t_end = c.t_end;
    const int w = c.w, lane = c.lane, g = c.g, t4 = c.t4, b0 = c.b0, b1 = c.b1;
    const bool v0 = c.v0, v1 = c.v1;
    const float* gbias = c.gbias;
    int* ys = c.ys;
    unsigned long long* trc = c.trc;
    const int tr_t = c.tr_t;
    if (w == NCW) {
        if (lane == 0) {
            uint32_t pc = 0;
            auto put = [&](const unsigned char* src, uint32_t bytes) {
                const uint32_t sl = pc % M::NSLOT1;
                mbar_wait(s_empty + 8 * sl, ((pc / M::NSLOT1) & 1) ^ 1);
                mbar_arrive_expect_tx(s_full + 8 * sl, bytes);
                tma_load_1d(sm + M::T_RING + sl * M::SLOT1, src, bytes, s_full + 8 * sl);
                pc++;
            };
            for (int t = t_begin; t < t_end; t++)
                for (int l = 0; l < L; l++) put(img + (size_t)l * im.layer_bytes + C::W_SKIP, S * 128);
        }
    } else if (w < NCW) {
        const float* s_bout = reinterpret_cast<const float*>(smem_raw + M::T_BOUT);
        const uint32_t o_skip = (uint32_t)(w * C::NSK * 2) * 512 + lane16;
        uint4 zsw[2][S / 32];
        load_out_w<S, TR>(c, zsw, 0);
        float sk[C::NSK][4];
#pragma unroll
        for (int i = 0; i < C::NSK; i++) sk[i][0] = sk[i][1] = sk[i][2] = sk[i][3] = 0.f;
        uint32_t pc = 0, hcnt = 0;
        for (int t = t_begin; t < t_end; t++) {
            constexpr int RPW = M::RPW;
            float sel[RPW];                                   // selectors of this warp's rows ub + RPW w + r
#pragma unroll
            for (int r = 0; r < RPW; r++) sel[r] = (ub + RPW * w + r) < B ? p.sel[(size_t)t * B + ub + RPW * w + r] : 0.5f;
            for (int l = 0; l < L; l++, pc++, hcnt++) {
                const uint32_t hb = sm + M::T_HBUF + (hcnt % M::NHB) * M::XT;
                mbar_wait(s_hfull + 8 * (hcnt % M::NHB), (hcnt / M::NHB) & 1);
                TRACE2(1, 16);
                uint32_t ha[4][4];
#pragma unroll
                for (int j = 0; j < 4; j++) load_a_rows<TR>(ha[j], hb, j, lane);
                const uint32_t sl = pc % M::NSLOT1, p2 = sm + M::T_RING + sl * M::SLOT1;
                mbar_wait(s_full + 8 * sl, (pc / M::NSLOT1) & 1);
#pragma unroll
                for (int jp = 0; jp < 2; jp++) {
                    uint4 bw[C::NSK];
#pragma unroll
                    for (int i = 0; i < C::NSK; i++) bw[i] = lds128(p2 + o_skip + (i * 2 + jp) * 512);
#pragma unroll
                    for (int i = 0; i < C::NSK; i++) hmma(sk[i], ha[2 * jp], bw[i].x, bw[i].y);
#pragma unroll
                    for (int i = 0; i < C::NSK; i++) hmma(sk[i], ha[2 * jp + 1], bw[i].z, bw[i].w);
                }
                // the h tile has been read (the HMMAs above hold its values): arm its barrier for the tile after next (one thread,
                // ordered before this warp's "free" signal), then hand the buffer back to the chain CTA
                if (tid == 0) mbar_arrive_expect_tx(s_hfull + 8 * (hcnt % M::NHB), M::XT);
                release_remote(s_hfree + 8 * (hcnt % M::NHB), 0, lane);
                release(s_empty + 8 * sl, lane);
                TRACE2(1, 15);
                if (DUMP) {
                    const float* pre = gbias + im.b_skpre + (size_t)l * S;
#pragma unroll
                    for (int i = 0; i < C::NSK; i++) {
                        const int c = 8 * (w * C::NSK + i) + 2 * t4;
                        float o0 = sk[i][0] + pre[c], o1 = sk[i][1] + pre[c + 1], o2 = sk[i][2] + pre[c], o3 = sk[i][3] + pre[c + 1];
                        if (l == L - 1) { o0 = fmaxf(o0, 0.f); o1 = fmaxf(o1, 0.f); o2 = fmaxf(o2, 0.f); o3 = fmaxf(o3, 0.f); }
                        if (v0) { p.skipOut[((size_t)l * B + b0) * S + c] = o0; p.skipOut[((size_t)l * B + b0) * S + c + 1] = o1; }
                        if (v1) { p.skipOut[((size_t)l * B + b1) * S + c] = o2; p.skipOut[((size_t)l * B + b1) * S + c + 1] = o3; }
                    }
                }
            }
            // ---------------- relu(skip + bias) -> Zs -> Za   (reference.cpp:93-104)
            {   // relu(skip + Bskip): TR bytes per pair of skip n-tiles, into this CTA's OB0 and the prep CTA's (free once the
                // prep's warps have read the previous sample's)
                uint4 v[C::NSK / 2];
#pragma unroll
                for (int i = 0; i < C::NSK; i++) {
                    uint32_t lo, hi;
                    relu_skip(sk[i], s_bout, 8 * (w * C::NSK + i) + 2 * t4, lo, hi);
                    if (i & 1) { v[i >> 1].z = lo; v[i >> 1].w = hi; } else { v[i >> 1].x = lo; v[i >> 1].y = hi; }
                }
                mbar_wait(s_ob0free, ((uint32_t)(t - t_begin) & 1) ^ 1);
                const uint32_t r_ob0full = mapa_u32(s_ob0full, 2);
#pragma unroll
                for (int j = 0; j < C::NSK / 2; j++) {
                    const uint32_t o = (uint32_t)((w * C::NSK / 2 + j) * 32 * TR + lane * TR);
                    if (TR == TU) {
                        sts128(sm + M::T_OB0 + o, v[j]);
                        st_async_v4(mapa_u32(sm + M::P_OB0 + o, 2), v[j], r_ob0full);
                    } else {                               // rows g: a0 a2
                        sts64(sm + M::T_OB0 + o, v[j].x, v[j].z);
                        st_async_v2(mapa_u32(sm + M::P_OB0 + o, 2), v[j].x, v[j].z, r_ob0full);
                    }
                }
            }
            bar_compute();
            TRACE2(1, 20);
            float zz[2][4];
            out_half<S, TR, DUMP, TRC>(c, trn, t, zsw, 0, zz);
#pragma unroll
            for (int i = 0; i < 2; i++) {
                const int c = 8 * (2 * w + i) + 2 * t4;
                sts64(sm + M::T_LBUF + (g * LROW + c) * 4, __float_as_uint(zz[i][0]), __float_as_uint(zz[i][1]));
                if (TR == TU) sts64(sm + M::T_LBUF + ((g + 8) * LROW + c) * 4, __float_as_uint(zz[i][2]), __float_as_uint(zz[i][3]));
            }
            bar_compute();
            mbar_wait(s_lfull, (uint32_t)(t - t_begin) & 1);  // columns 128-255 from the prep CTA
            TRACE2(1, 22);
            {   // softmax + categorical sample: warp w serves utterances RPW w .. RPW w + RPW - 1 of the tile (two of 16, one of 8);
                // lane holds 8 consecutive classes of each
                float e[RPW][8], m[RPW];
#pragma unroll
                for (int r = 0; r < RPW; r++) {
                    const uint4 u0 = lds128(sm + M::T_LBUF + ((RPW * w + r) * LROW + 8 * lane) * 4), u1 = lds128(sm + M::T_LBUF + ((RPW * w + r) * LROW + 8 * lane + 4) * 4);
                    e[r][0] = __uint_as_float(u0.x); e[r][1] = __uint_as_float(u0.y); e[r][2] = __uint_as_float(u0.z); e[r][3] = __uint_as_float(u0.w);
                    e[r][4] = __uint_as_float(u1.x); e[r][5] = __uint_as_float(u1.y); e[r][6] = __uint_as_float(u1.z); e[r][7] = __uint_as_float(u1.w);
                    m[r] = e[r][0];                           // the row's own logits, not 0 as in the CPU model: see lat_compute
#pragma unroll
                    for (int k = 1; k < 8; k++) m[r] = fmaxf(m[r], e[r][k]);
                }
#pragma unroll
                for (int o = 16; o >= 1; o >>= 1) {
#pragma unroll
                    for (int r = 0; r < RPW; r++) m[r] = fmaxf(m[r], __shfl_xor_sync(0xffffffffu, m[r], o));
                }
                // the logits have been read: arm lfull for the prep's next half, then hand the buffer back to it
                if (tid == 0) mbar_arrive_expect_tx(s_lfull, TR * 128 * 4);
                release_remote(s_lfree, 2, lane);
                float incl[RPW], tot_lane[RPW];
#pragma unroll
                for (int r = 0; r < RPW; r++) {
                    const float ms = m[r] * 1.4426950408889634f;
                    float run = 0.f;
#pragma unroll
                    for (int k = 0; k < 8; k++) { run += wn::exp2f_fast(fmaf(e[r][k], 1.4426950408889634f, -ms)); e[r][k] = run; }
                    incl[r] = tot_lane[r] = run;
                }
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    float a[RPW];
#pragma unroll
                    for (int r = 0; r < RPW; r++) a[r] = __shfl_up_sync(0xffffffffu, incl[r], o);
                    if (lane >= o) {
#pragma unroll
                        for (int r = 0; r < RPW; r++) incl[r] += a[r];
                    }
                }
                int yv[RPW];                                  // the sampled index of each row
#pragma unroll
                for (int r = 0; r < RPW; r++) {
                    const float total = __shfl_sync(0xffffffffu, incl[r], 31);
                    const float excl = incl[r] - tot_lane[r];
                    const float target = sel[r] * total;
                    int cntk = 0;
#pragma unroll
                    for (int k = 0; k < 8; k++) cntk += (target < excl + e[r][k]) ? 0 : 1;
                    const unsigned ball = __ballot_sync(0xffffffffu, target < incl[r]);
                    const int lf = ball ? __ffs(ball) - 1 : 31;
                    const int ck = __shfl_sync(0xffffffffu, cntk, lf);
                    yv[r] = ball ? 8 * lf + (ck < 7 ? ck : 7) : A - 1;
                    const int b = ub + RPW * w + r;
                    if (DUMP && b < B) {
                        const float inv = 1.f / total;
                        float prevv = 0.f;
#pragma unroll
                        for (int k = 0; k < 8; k++) { p.P[(size_t)b * A + 8 * lane + k] = (e[r][k] - prevv) * inv; prevv = e[r][k]; }
                    }
                }
                // both rows' indices are chosen before lane 0 stores anything: the shuffles of the second row cannot move past the
                // first row's stores, so selecting and storing row by row would run the two selections one after the other
                if (lane == 0) {
                    int fbk[RPW], yold[RPW];
#pragma unroll
                    for (int r = 0; r < RPW; r++) {
                        const int b = ub + RPW * w + r;
                        fbk[r] = yv[r];
                        if (b < B) {
                            p.yOut[(size_t)b * p.N + t] = yv[r];
                            if (p.forced) fbk[r] = p.forced[(size_t)b * p.N + t];
                        } else fbk[r] = 128;
                        yold[r] = ys[RPW * w + r];
                        ys[TR + RPW * w + r] = yold[r];
                        ys[RPW * w + r] = fbk[r];
                    }
                    if (t + 1 < t_end) {                      // the chain CTA's copy: data + completion on its yfull barrier
                        const uint32_t rb = mapa_u32(s_yfull, 0);
                        const uint32_t ryold = mapa_u32(sm + M::O_YS + (TR + RPW * w) * 4, 0), rycur = mapa_u32(sm + M::O_YS + (RPW * w) * 4, 0);
                        if (RPW == 2) {
                            st_async_v2(ryold, (uint32_t)yold[0], (uint32_t)yold[RPW - 1], rb);
                            st_async_v2(rycur, (uint32_t)fbk[0], (uint32_t)fbk[RPW - 1], rb);
                        } else {
                            st_async_b32(ryold, (uint32_t)yold[0], rb);
                            st_async_b32(rycur, (uint32_t)fbk[0], rb);
                        }
                    }
                }
            }
            TRACE2(1, 23);
            bar_compute();
        }
        store_ys<TR>(p, B, ys, ub, tid);
    }
}

// ===================================================================================== prep CTA
// (Bh + Lh) + Wprev . x[t-d] of every step, as far ahead of the chain CTA as its NAP tile buffers allow.  Nothing here depends on
// the current sample: the history it reads was written by the chain CTA at least L - 9 steps earlier (wn_launch_lat asks for L >= 12).
template <int S, int TR, bool DUMP, bool TRC, bool WIDE>
__device__ __forceinline__ void prep_cta(const ClusterCta& c, int& trn)
{
    using C = Cfg<S>;
    using M = CfgC<S, TR>;
    const WnParams& p = c.p;
    const unsigned char* img = c.img;
    const LatImage& im = c.im;
    unsigned char* smem_raw = c.smem;
    const uint32_t sm = c.sm, hw4 = c.hw4, lane16 = c.lane16;
    const uint32_t s_full = c.s_full, s_empty = c.s_empty, s_pfull = c.s_pfull, s_apfull = c.s_apfull, s_apfree = c.s_apfree;
    const uint32_t s_lfull = c.s_lfull, s_lfree = c.s_lfree;
    const int L = c.L, tid = c.tid, tile = c.tile, slots = c.slots, t_begin = c.t_begin, t_end = c.t_end, ntiles_alloc = c.ntiles_alloc;
    const int w = c.w, lane = c.lane, g = c.g, t4 = c.t4;
    unsigned long long* trc = c.trc;
    const int tr_t = c.tr_t;
    const int nsteps = p.count * L;
    if (w == NCW) {
        if (lane == 0) {
            int l = 0;
            for (int n = 0; n < nsteps; n++) {
                const uint32_t sl = (uint32_t)n % M::NPRING;
                mbar_wait(s_empty + 8 * sl, (((uint32_t)n / M::NPRING) & 1) ^ 1);
                mbar_arrive_expect_tx(s_full + 8 * sl, 16384);
                // Wprev of layer l lives in the block of the layer before it (lat_pack_kernel)
                tma_load_1d(sm + M::P_RING + sl * 16384, img + (size_t)((l + L - 1) % L) * im.layer_bytes + C::W_PREV, 16384, s_full + 8 * sl);
                if (++l == L) l = 0;
            }
        }
    } else if (w < NCW) {
        int* dil = reinterpret_cast<int*>(smem_raw + M::P_DIL);
        const uint32_t rstride = (uint32_t)ntiles_alloc * 2048u, cstride = (uint32_t)ntiles_alloc * 4096u;
        const unsigned char* gring = static_cast<const unsigned char*>(p.ring) + (size_t)tile * 2048;
        const uint32_t o_t0 = (uint32_t)(w * 2) * 512 + lane16, o_g0 = (uint32_t)((8 + w) * 2) * 512 + lane16;
        const uint32_t r_ap = mapa_u32(sm + M::C_AP + (uint32_t)tid * (2 * TR), 0);   // this thread's 2 TR / 4 floats of the chain CTA's tiles
        const uint32_t r_apfull = mapa_u32(s_apfull, 0);
        const uint32_t s_cond = sm + M::P_COND + (uint32_t)tid * 16;              // this thread's 16 B of a conditioning tile (+ 4 KB per slot)
        const uint32_t s_bias = sm + M::P_BIAS + (uint32_t)(w * 4 + t4) * 16;     // this thread's Bh of layer 0 (+ 512 B per layer)
        // Staging of the step `itp`, three steps before its use, no register and no scoreboard involved:
        //  * its conditioning tile: every thread copies the 16 bytes it will read back itself (cp.async; completion = the thread's
        //    own cp.async group, no barrier);
        //  * its dilated history x_l[t-d] (zero before the start of the utterance, nv_wavenet.cuh:106): warps 0-3, 128 x 16 B,
        //    completion on an mbarrier (every warp reads the whole tile).
        // Both are copied as whole 16-byte groups of the 16-row store layouts with cp.async.cg, which bypasses L1, at either tile
        // height; an 8-row tile picks its rows' words when it reads them back (own_rows).  The history ring is rewritten during the
        // launch by the chain CTA on another SM with plain stores, and L1 is not coherent across SMs: a narrower copy through L1
        // (cp.async.ca, the only form below 16 bytes) could find the line of the slot's previous occupant, maxDil + 1 samples old.
        // NPS = 8 slots: a slot is staged again five steps after its use, and the weight ring (NPRING = 4 pieces) keeps the warps within four.
        // itp.t counts the (clamped) absolute time of the WnParams, so the test against d is the utterance's.
        StepIt itp{p.hist_t, 0, p.ring_slot};
        const int h_end = p.hist_t + p.count;
        uint32_t pcnt = 0;
        const unsigned char* cptr = static_cast<const unsigned char*>(p.Lh) + (size_t)tile * 4096 + (size_t)(w * 32 + lane) * 16 + (size_t)t_begin * L * cstride;
        auto stage = [&]() {
            const uint32_t slot = pcnt % M::NPS;
            if (itp.t < h_end) cp_async16(s_cond + slot * 4096, cptr);
            cptr += cstride;
            if (w < 4) {
                const int d = dil[itp.l];
                const uint32_t dst = sm + M::P_PST + slot * 2048 + (uint32_t)(w * 32 + lane) * 16;
                if (itp.t >= h_end || itp.t < d) {
                    sts128(dst, make_uint4(0, 0, 0, 0));
                    mbar_arrive(s_pfull + 8 * slot);
                } else {
                    int sl = itp.slot - d; if (sl < 0) sl += slots;
                    cp_async16(dst, gring + ring_off<WIDE>(sl * L + itp.l, rstride) + (size_t)(w * 32 + lane) * 16);
                    cp_async_arrive_noinc(s_pfull + 8 * slot);
                }
            }
            cp_async_commit();
            pcnt++;
            if (++itp.l == L) { itp.l = 0; itp.t++; if (++itp.slot == slots) itp.slot = 0; }
        };
        uint4 zsw[2][S / 32];
        load_out_w<S, TR>(c, zsw, 1);
        // output columns 128-255 of sample t; the logits go to the tail CTA (free once its softmax has read the previous ones)
        auto out_prep = [&](const int t) {
            float zz[2][4];
            TRACE2(2, 30);
            out_half<S, TR, DUMP, TRC>(c, trn, t, zsw, 1, zz);
            const uint32_t r_lfull = mapa_u32(s_lfull, 1);
            mbar_wait(s_lfree, ((uint32_t)(t - t_begin) & 1) ^ 1);
#pragma unroll
            for (int i = 0; i < 2; i++) {
                const int c = 8 * (16 + 2 * w + i) + 2 * t4;
                st_async_v2(mapa_u32(sm + M::T_LBUF + (g * LROW + c) * 4, 1), __float_as_uint(zz[i][0]), __float_as_uint(zz[i][1]), r_lfull);
                if (TR == TU) st_async_v2(mapa_u32(sm + M::T_LBUF + ((g + 8) * LROW + c) * 4, 1), __float_as_uint(zz[i][2]), __float_as_uint(zz[i][3]), r_lfull);
            }
            TRACE2(2, 33);
        };
        stage(); stage(); stage();
        int l1 = 0, tout = t_begin;                        // tout: the next sample whose output half is due
        for (int n = 0; n < nsteps; n++) {
            const uint32_t sl = (uint32_t)n % M::NPRING, pa = sm + M::P_RING + sl * 16384, slot = (uint32_t)n % M::NPS, buf = (uint32_t)n % M::NAP;
            cp_async_wait_pending<2>();                    // this thread's conditioning of step n has landed (two later groups may be in flight)
            // (tanh, tanh, sigmoid, sigmoid) of rows (g, g + 8, g, g + 8); 8-row tiles: (tanh, 0, sigmoid, 0) of their row
            const uint4 cb = own_rows<TR>(lds128(s_cond + slot * 4096), hw4 != 0);
            const uint4 bq = lds128(s_bias + l1 * 512);
            mbar_wait(s_full + 8 * sl, ((uint32_t)n / M::NPRING) & 1);
            const GateW bw = lds_gate_w(pa, o_t0, o_g0);
            mbar_wait(s_pfull + 8 * slot, ((uint32_t)n / M::NPS) & 1);
            uint32_t pb[4][4];
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const uint4 v = own_rows<TR>(lds128(sm + M::P_PST + slot * 2048 + j * 512 + lane16), hw4 != 0);
                pb[j][0] = v.x; pb[j][1] = v.y; pb[j][2] = v.z; pb[j][3] = v.w;
            }
            const float4 bh = make_float4(__uint_as_float(bq.x), __uint_as_float(bq.y), __uint_as_float(bq.z), __uint_as_float(bq.w));
            const float2 c0 = unpack_h2(cb.x), c1 = unpack_h2(cb.y), c2 = unpack_h2(cb.z), c3 = unpack_h2(cb.w);
            float a[2][4] = {{bh.x + c0.x, bh.y + c0.y, bh.x + c1.x, bh.y + c1.y}, {bh.z + c2.x, bh.w + c2.y, bh.z + c3.x, bh.w + c3.y}};
            float u[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
            hmma_k64(a, u, pb, bw);
            release(s_empty + 8 * sl, lane);
            // the chain CTA's tile buffer n % NAP is free once it has read tile n - NAP
            mbar_wait(s_apfree + 8 * buf, ((n / M::NAP) & 1) ^ 1);
            if (TR == TU) {
                st_async_v4(r_ap + buf * M::AP, a[0][0] + u[0][0], a[0][1] + u[0][1], a[0][2] + u[0][2], a[0][3] + u[0][3], r_apfull + 8 * buf);
                st_async_v4(r_ap + buf * M::AP + 16, a[1][0] + u[1][0], a[1][1] + u[1][1], a[1][2] + u[1][2], a[1][3] + u[1][3], r_apfull + 8 * buf);
            } else {                                       // row g: tanh pair, sigmoid pair
                st_async_v4(r_ap + buf * M::AP, a[0][0] + u[0][0], a[0][1] + u[0][1], a[1][0] + u[1][0], a[1][1] + u[1][1], r_apfull + 8 * buf);
            }
            stage();
            if (++l1 == L) l1 = 0;
            // the output half of sample tout: after step (tout + 1, 1) has been shipped, so that the chain CTA starts sample
            // tout + 1 with its first two pre-activation tiles at hand, and before the wait for the buffer of step
            // (tout + 1, NAP + 1), which the chain CTA frees only inside sample tout + 1
            if (n == (tout - t_begin + 1) * L + 1) out_prep(tout++);
        }
        while (tout < t_end) out_prep(tout++);             // the last sample: no steps follow it
        cp_async_wait_all();
    }
}

// MODELS: p.group_model is set, and the cluster's weights are its group's model's (DESIGN.md §6).
// WIDE: the history ring passes 4 GiB, and its offsets are formed in 64 bits (ring_off).
template <int S, int TR, bool DUMP, bool TRC, bool MODELS, bool WIDE>
__global__ void __launch_bounds__(NTC, 1) wn_lat2_kernel(const WnParams p, const unsigned char* __restrict__ img0, const int ntiles_alloc)
{
    // debug timeline (tools/lat_trace.py, TRACE2): role = cluster rank (0 chain, 1 tail, 2 prep), thread 0 of each CTA of the first cluster
    unsigned long long* trc = (TRC && p.trace && blockIdx.x < NCL) ? p.trace : nullptr;
    int trn = 0;
    const int tr_t = p.trace_t & 0xFFFF;
    using C = Cfg<S>;
    using M = CfgC<S, TR>;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const uint32_t sm = smem_u32(smem_raw);
    const int L = p.L, B = p.B;
    const LatImage im = lat_image(S, L);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    uint32_t crank;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(crank));
    const bool is_chain = crank == 0, is_tail = crank == 1;
    // this cluster serves utterances ub .. ub + TR - 1: all of 16-row tile `tile` of the conditioning store and the history ring, or
    // (TR = 8) its half ub & 8, whose words sit `hw4` bytes into every 16-byte group of the tile's accumulator / A-fragment order
    const int ub = blockIdx.x / NCL * TR, tile = ub / TU;
    const WnGroupWeights gw = MODELS ? wn_group_weights(p, ub) : WnGroupWeights{0, img0};
    const unsigned char* __restrict__ img = gw.image;
    const uint32_t hw4 = (uint32_t)(ub & 8) >> 1;
    const int slots = p.maxDil + 1;
    const int t_begin = p.init_sample, t_end = p.init_sample + p.count;
    const float* gbias = reinterpret_cast<const float*>(img + im.off_bias);

    // barriers (same offsets in every CTA): ring full[NRING] / empty[NRING] (the chain uses NSLOT0 of each, the tail NSLOT1, the prep NPRING);
    // pfull[NPS] (prep: staged history tiles); hfull[NHB] (tail: h tiles, bytes from the chain); hfree[NHB], yfull, apfull[NAP] (chain: bytes from the tail / the prep CTA);
    // apfree[NAP] (prep: arrived by the chain's warps).  Output layers, once per sample: ob0full (prep: relu(skip) bytes from the
    // tail); ob0free (tail: arrived by the prep's warps); ob1full (tail and prep: the peer's relu(Zs) half); ob1free (tail and prep:
    // arrived by the warps of both CTAs once they have read OB1); lfull (tail: the prep's logits bytes); lfree (prep: arrived by the
    // tail's warps once the softmax has read the logits)
    const uint32_t bar = sm + M::O_BAR;
    const uint32_t s_full = bar + M::B_FULL, s_empty = bar + M::B_EMPTY, s_pfull = bar + M::B_PFULL, s_hfull = bar + M::B_HFULL, s_hfree = bar + M::B_HFREE;
    const uint32_t s_yfull = bar + M::B_YFULL, s_apfull = bar + M::B_APFULL, s_apfree = bar + M::B_APFREE;
    const uint32_t s_ob0full = bar + M::B_OB0FULL, s_ob0free = bar + M::B_OB0FREE, s_ob1full = bar + M::B_OB1FULL, s_ob1free = bar + M::B_OB1FREE;
    const uint32_t s_lfull = bar + M::B_LFULL, s_lfree = bar + M::B_LFREE;
    int* ys = reinterpret_cast<int*>(smem_raw + M::O_YS);

    if (tid == 0) {
        for (int i = 0; i < M::NRING; i++) { mbar_init(s_full + 8 * i, 1); mbar_init(s_empty + 8 * i, is_chain ? 1 : NCW); }
        for (int i = 0; i < M::NPS; i++) mbar_init(s_pfull + 8 * i, 128);
        for (int i = 0; i < M::NHB; i++) { mbar_init(s_hfull + 8 * i, 1); mbar_init(s_hfree + 8 * i, NCW); }
        for (int i = 0; i < M::NAP; i++) { mbar_init(s_apfull + 8 * i, 1); mbar_init(s_apfree + 8 * i, 1); }
        mbar_init(s_yfull, 1);
        mbar_init(s_ob0full, 1); mbar_init(s_ob0free, NCW); mbar_init(s_ob1full, 1); mbar_init(s_ob1free, 2 * NCW);
        mbar_init(s_lfull, 1); mbar_init(s_lfree, NCW);
        fence_mbar_init();
        // transaction barriers are armed by their owner one phase ahead: the tail expects an h tile per step (TR x 128 B), the chain
        // the sampled indices (2 x TR x 4 B) and a pre-activation tile per step (TR x 512 B); once per sample the prep expects relu(skip)
        // and a relu(Zs) half, the tail a relu(Zs) half and the logits half
        if (is_chain) { mbar_arrive_expect_tx(s_yfull, 2 * TR * 4); for (int i = 0; i < M::NAP; i++) mbar_arrive_expect_tx(s_apfull + 8 * i, M::AP); }
        else if (is_tail) {
            for (int i = 0; i < M::NHB; i++) mbar_arrive_expect_tx(s_hfull + 8 * i, M::XT);
            mbar_arrive_expect_tx(s_ob1full, TR * 128 * 2); mbar_arrive_expect_tx(s_lfull, TR * 128 * 4);
        }
        else { mbar_arrive_expect_tx(s_ob0full, TR * S * 2); mbar_arrive_expect_tx(s_ob1full, TR * 128 * 2); }
    }
    if (tid < TR) {
        const int b = ub + tid;
        ys[tid] = b < B ? p.yCur[b] : 128;
        ys[TR + tid] = b < B ? p.yPrev[b] : 128;
    }
    if (is_chain) {
        const uint32_t* ec = gw.at<uint32_t>(p.embCur);
        for (int i = tid; i < A * 32; i += NTC) sts32(sm + M::C_EMB + ((i >> 5) * EROW + (i & 31)) * 4, ec[i]);
        for (int i = tid; i < L * 256; i += NTC) sts32(sm + M::C_BIAS + i * 4, __float_as_uint(gbias[im.b_layer + i]));
    } else if (is_tail) {
        float* s_bout = reinterpret_cast<float*>(smem_raw + M::T_BOUT);
        for (int i = tid; i < S; i += NTC) s_bout[i] = gbias[im.b_skpre + (size_t)(L - 1) * S + i];
        for (int i = tid; i < A; i += NTC) { s_bout[S + i] = gbias[im.b_bzs + i]; s_bout[S + A + i] = gbias[im.b_bza + i]; }
    } else {
        int* dil = reinterpret_cast<int*>(smem_raw + M::P_DIL);
        if (tid == 0) { int d = 1; for (int l = 0; l < L; l++) { dil[l] = d; d <<= 1; if (d > p.maxDil) d = 1; } }   // nv_wavenet.cuh:99-111
        for (int i = tid; i < L * 128; i += NTC) sts32(sm + M::P_BIAS + i * 4, __float_as_uint(gbias[im.b_layer + (i >> 2) * 8 + (i & 3)]));
        float* s_bout = reinterpret_cast<float*>(smem_raw + M::P_BOUT);
        for (int i = tid; i < A; i += NTC) { s_bout[i] = gbias[im.b_bzs + i]; s_bout[A + i] = gbias[im.b_bza + i]; }
    }
    __syncthreads();
    cluster_sync_all();                                    // every CTA's barriers are initialised before anybody signals a peer

    const int w = warp, g = lane >> 2, t4 = lane & 3;
    const int b0 = ub + g, b1 = TR == TU ? b0 + 8 : B;       // an 8-row tile has no row g + 8
    const bool v0 = b0 < B, v1 = b1 < B;
    const uint32_t lane16 = (uint32_t)lane * 16;
    const uint32_t xchg = xslot<TR>(w, lane);                // this thread's slot of an activation tile
    const ClusterCta c{p, img, gw.at<void>(p.embPrev), im, smem_raw, sm, L, B, tid, crank, ub, tile, hw4, slots, t_begin, t_end, ntiles_alloc, gbias,
                       s_full, s_empty, s_pfull, s_hfull, s_hfree, s_yfull, s_apfull, s_apfree, s_ob0full, s_ob0free, s_ob1full, s_ob1free, s_lfull, s_lfree,
                       ys, w, lane, g, t4, b0, b1, v0, v1, lane16, xchg, trc, tr_t};
    if (is_chain) chain_cta<S, TR, DUMP, TRC, WIDE>(c, trn);
    else if (is_tail) tail_cta<S, TR, DUMP, TRC>(c, trn);
    else prep_cta<S, TR, DUMP, TRC, WIDE>(c, trn);
    // nobody leaves while the peer may still write into this CTA's shared memory or arrive on its barriers
    cluster_sync_all();
}
#undef TRACE2

}  // namespace

// ------------------------------------------------------------------------------------------------ host side
bool wn_lat_supported(int R_, int S, int A_, int L)
{
    return R_ == R && A_ == A && (S == 128 || S == 256) && L >= 4 && L <= MAXL;     // L >= 4: history prefetch runs 3 steps ahead (single-CTA kernel)
}
static size_t image_bytes(const WnConfig& c) { return lat_image(c.S, c.L).total; }

static cudaError_t cond_convert(const WnConfig& c, void* dst, const float* src_dev, int first_sample, int nsamples, cudaStream_t stream)
{
    return wn_layout_launch(lat_cond_kernel, (size_t)nsamples * c.L * lat_tiles(c.B) * 256, stream, c, static_cast<unsigned char*>(dst), src_dev,
                            first_sample);
}

static cudaError_t wn_lat_pack(void* image, const WnParams& p, cudaStream_t stream)
{
    const LatImage im = lat_image(p.S, p.L);
    cudaError_t e = cudaMemsetAsync(image, 0, im.total, stream);
    if (e != cudaSuccess) return e;
    lat_pack_kernel<<<296, 256, 0, stream>>>(p, static_cast<unsigned char*>(image), im);
    return cudaGetLastError();
}

// one launch of a latency kernel variant; p.B = utterances of this run, ntiles_alloc = tiles of the batch size the conditioning
// store / history ring were laid out for
using LatGo = cudaError_t (*)(const WnParams& p, const unsigned char* im8, int tiles, int ntiles_alloc, cudaStream_t stream);

template <int S, bool DUMP, bool TRC, bool MODELS, bool WIDE>
static cudaError_t lat_go(const WnParams& p, const unsigned char* im8, int tiles, int ntiles_alloc, cudaStream_t stream)
{
    const size_t smem = Cfg<S>::SMEM;
    const cudaError_t e = cudaFuncSetAttribute(wn_lat_kernel<S, DUMP, TRC, MODELS, WIDE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    wn_lat_kernel<S, DUMP, TRC, MODELS, WIDE><<<tiles, NT, smem, stream>>>(p, im8, ntiles_alloc);
    return cudaGetLastError();
}

// the cluster variant: grid = NCL x `clusters` CTAs, cluster (NCL, 1, 1); `at` receives the cluster attribute the config points to
template <int S, int TR>
static cudaLaunchConfig_t lat2_config(int clusters, cudaStream_t stream, cudaLaunchAttribute& at)
{
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(NCL * clusters, 1, 1);
    cfg.blockDim = dim3(NTC, 1, 1);
    cfg.dynamicSmemBytes = CfgC<S, TR>::SMEM;
    cfg.stream = stream;
    at.id = cudaLaunchAttributeClusterDimension;
    at.val.clusterDim.x = NCL; at.val.clusterDim.y = 1; at.val.clusterDim.z = 1;
    cfg.attrs = &at;
    cfg.numAttrs = 1;
    return cfg;
}
template <int S, int TR, bool DUMP, bool TRC, bool MODELS, bool WIDE>
static cudaError_t lat2_go(const WnParams& p, const unsigned char* im8, int clusters, int ntiles_alloc, cudaStream_t stream)
{
    cudaError_t e = cudaFuncSetAttribute(wn_lat2_kernel<S, TR, DUMP, TRC, MODELS, WIDE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CfgC<S, TR>::SMEM);
    if (e != cudaSuccess) return e;
    cudaLaunchAttribute at;
    const cudaLaunchConfig_t cfg = lat2_config<S, TR>(clusters, stream, at);
    e = cudaLaunchKernelEx(&cfg, wn_lat2_kernel<S, TR, DUMP, TRC, MODELS, WIDE>, p, im8, ntiles_alloc);
    return e != cudaSuccess ? e : cudaGetLastError();
}
// how many clusters the device runs at once (a cluster needs NCL SMs of one GPC: fewer than 132 / NCL fit on an H100); 0 if the query fails
template <int S, int TR>
static int lat2_max_clusters()
{
    static int cached = -1;
    if (cached >= 0) return cached;
    if (cudaFuncSetAttribute(wn_lat2_kernel<S, TR, false, false, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CfgC<S, TR>::SMEM) != cudaSuccess) { cudaGetLastError(); return cached = 0; }
    cudaLaunchAttribute at;
    const cudaLaunchConfig_t cfg = lat2_config<S, TR>(48, 0, at);
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, wn_lat2_kernel<S, TR, false, false, false, false>, &cfg) != cudaSuccess) { cudaGetLastError(); n = 0; }
    return cached = n;
}

// a dumping launch = every sample but the last with the plain (or tracing) variant, then the last one with the dumping variant
// (a continuation is bit-identical to one launch: the whole state lives in global memory between launches)
static cudaError_t lat_launch_split(const WnParams& p, LatGo plain, LatGo trace, LatGo dump, const unsigned char* im8, int tiles, int ntiles_alloc,
                                    cudaStream_t stream)
{
    WnParams head = p, tail = p;
    if (p.dump) { head.count = p.count - 1; head.dump = 0; tail = wn_params_skip(p, p.count - 1); }
    cudaError_t e = cudaSuccess;
    if (head.count > 0) e = (p.trace ? trace : plain)(head, im8, tiles, ntiles_alloc, stream);
    if (e == cudaSuccess && p.dump) e = dump(tail, im8, tiles, ntiles_alloc, stream);
    return e;
}
template <int S, bool WIDE>
static cudaError_t lat_launch_W(const WnParams& p, const unsigned char* im8, int tiles, int ntiles_alloc, cudaStream_t stream)
{
    if (p.group_model)
        return lat_launch_split(p, lat_go<S, false, false, true, WIDE>, lat_go<S, false, true, true, WIDE>, lat_go<S, true, false, true, WIDE>, im8, tiles,
                                ntiles_alloc, stream);
    return lat_launch_split(p, lat_go<S, false, false, false, WIDE>, lat_go<S, false, true, false, WIDE>, lat_go<S, true, false, false, WIDE>, im8, tiles,
                            ntiles_alloc, stream);
}
template <int S>
static cudaError_t lat_launch_S(const WnParams& p, const unsigned char* im8, int tiles, int ntiles_alloc, cudaStream_t stream, size_t* smem_out)
{
    *smem_out = Cfg<S>::SMEM;
    return lat_ring_wide(p.maxDil, p.L, ntiles_alloc) ? lat_launch_W<S, true>(p, im8, tiles, ntiles_alloc, stream)
                                                      : lat_launch_W<S, false>(p, im8, tiles, ntiles_alloc, stream);
}
template <int S, int TR, bool WIDE>
static cudaError_t lat2_launch_W(const WnParams& p, const unsigned char* im8, int clusters, int ntiles_alloc, cudaStream_t stream)
{
    if (p.group_model)
        return lat_launch_split(p, lat2_go<S, TR, false, false, true, WIDE>, lat2_go<S, TR, false, true, true, WIDE>, lat2_go<S, TR, true, false, true, WIDE>, im8,
                                clusters, ntiles_alloc, stream);
    return lat_launch_split(p, lat2_go<S, TR, false, false, false, WIDE>, lat2_go<S, TR, false, true, false, WIDE>, lat2_go<S, TR, true, false, false, WIDE>,
                            im8, clusters, ntiles_alloc, stream);
}
template <int S, int TR>
static cudaError_t lat2_launch_S(const WnParams& p, const unsigned char* im8, int clusters, int ntiles_alloc, cudaStream_t stream, size_t* smem_out)
{
    *smem_out = CfgC<S, TR>::SMEM;
    return lat_ring_wide(p.maxDil, p.L, ntiles_alloc) ? lat2_launch_W<S, TR, true>(p, im8, clusters, ntiles_alloc, stream)
                                                      : lat2_launch_W<S, TR, false>(p, im8, clusters, ntiles_alloc, stream);
}

template <int TR>
static int lat2_fit(int S) { return S == 256 ? lat2_max_clusters<256, TR>() : S == 128 ? lat2_max_clusters<128, TR>() : 0; }
int wn_lat_max_clusters(int S, int rows) { return rows == 8 ? lat2_fit<8>(S) : rows == TU ? lat2_fit<TU>(S) : 0; }

// c.lat_cluster: serve the utterances with clusters of three CTAs (chain / tail / prep) instead of one CTA per 16-utterance tile.
// A cluster takes 8 utterances while all of them are resident at once, else 16 (a second wave would halve the rate): an 8-row
// cluster does half the per-row work of a 16-row one (tile reads, gate, residual, output epilogues, softmax) on the same HMMAs and
// weight reads, so it is faster per utterance as long as there are SMs for twice the clusters.  A run of fewer utterances than the
// engine holds takes the first p.B of them: the conditioning store and the history ring stay laid out per 16-utterance tile of the
// engine's batch, whichever tile height runs.
// The utterances per cluster of a run of `batch` utterances: 8, 16 (TU), or 0 when the single-CTA kernel runs.
// The cluster kernel's prep CTA reads history tiles the chain CTA wrote at least L - 9 steps earlier: it wants a few steps of margin.
static int lat_cluster_rows(const WnConfig& c, int batch)
{
    if (!c.lat_cluster || c.L < 12 || (c.S != 256 && c.S != 128)) return 0;
    if ((batch + 7) / 8 <= lat2_fit<8>(c.S)) return 8;
    if (lat_tiles(batch) <= lat2_fit<TU>(c.S)) return TU;
    return 0;
}
// A model group is what a full-batch run serves per cluster when that is 8 rows, else a 16-row tile.  A smaller run's clusters lie
// inside these groups: fewer utterances never take a taller tile.
static int lat_group_rows(const WnConfig& c) { return lat_cluster_rows(c, c.B) == 8 ? 8 : TU; }

static cudaError_t wn_launch_lat(const WnConfig& c, const WnParams& p, const void* image, cudaStream_t stream, WnLaunchInfo* info)
{
    const int grid = lat_tiles(p.B), ntiles_alloc = lat_tiles(c.B);
    const unsigned char* im8 = static_cast<const unsigned char*>(image);
    size_t smem = 0;
    cudaError_t e;
    {
        const int tr = lat_cluster_rows(c, p.B), clusters = tr == 8 ? (p.B + 7) / 8 : grid;
        if (tr == 8) e = p.S == 256 ? lat2_launch_S<256, 8>(p, im8, clusters, ntiles_alloc, stream, &smem) : lat2_launch_S<128, 8>(p, im8, clusters, ntiles_alloc, stream, &smem);
        else if (tr == TU) e = p.S == 256 ? lat2_launch_S<256, TU>(p, im8, clusters, ntiles_alloc, stream, &smem) : lat2_launch_S<128, TU>(p, im8, clusters, ntiles_alloc, stream, &smem);
        if (tr) {
            if (e != cudaSuccess) return e;
            if (info) { info->kernel = NVWN_KERNEL_LATENCY; info->grid = NCL * clusters; info->block = NTC; info->smem_bytes = (int)smem; info->batch_per_cta = tr; info->cluster = NCL; }
            return cudaGetLastError();
        }
    }
    if (p.S == 256) e = lat_launch_S<256>(p, im8, grid, ntiles_alloc, stream, &smem);
    else if (p.S == 128) e = lat_launch_S<128>(p, im8, grid, ntiles_alloc, stream, &smem);
    else return cudaErrorInvalidValue;
    if (e != cudaSuccess) return e;
    if (info) { info->kernel = NVWN_KERNEL_LATENCY; info->grid = grid; info->block = NT; info->smem_bytes = (int)smem; info->batch_per_cta = TU; info->cluster = 1; }
    return cudaGetLastError();
}

const WnFamily wn_lat_family = {LatLayout::store_bytes, LatLayout::ring_bytes, image_bytes, cond_convert, wn_readback<LatLayout>,
                                wn_clear_rows<LatLayout>, wn_convert_rows<LatLayout>, wn_put_history<LatLayout>, wn_get_history<LatLayout>,
                                wn_put_history_rows<LatLayout>, wn_get_history_rows<LatLayout>, wn_clear_times<LatLayout>,
                                wn_lat_pack, wn_launch_lat, false, lat_group_rows};
