// wn_tc_kernel.cu -- fp16 tensor-core kernel of the WaveNet inference loop (sm_90a: wgmma + bulk TMA + mbarrier).
//
// ONE persistent CTA per 64 utterances runs the whole autoregressive loop for `count` samples.  Every GEMM of a
// layer is  D[64 utterances x N channels] (fp32, registers) (+)= X[64 x 64] . W[N x 64]^T  on the warpgroup MMA, activations
// as the A operand and weights as the B operand, both K-major SWIZZLE_128B tiles in shared memory.
//
//   warpgroups 0, 1  consumers.  Warpgroup w owns residual / gate channels [32 w, 32 w + 32) and the w-th half of the skip,
//                    Zs and Za columns of all 64 utterances, so that the gate (tanh(a_c) * sigmoid(g_c) needs accumulator
//                    columns c and 64 + c) and the residual update stay local to a thread of the accumulator fragment.
//                    They issue the MMAs and evaluate embedding -> per layer [gate -> h tile] [x += Wres.h + Bres -> x tile,
//                    history ring] -> relu(skip) tile -> relu(Zs) tile -> softmax + categorical sample.
//   warp 8           TMA producer.  Streams the pre-tiled fp16 weight image, the conditioning tiles and the x[t-d]
//                    history tiles from L2 through an NSTAGE x 16 KB shared-memory ring with cp.async.bulk + mbarrier
//                    complete_tx, in exactly the order the consumers take them.
//
// Tiles: the conditioning store and the history ring are laid out per tile of 64 utterances (default), 32 (the MMA rows of
// the other 32 stay empty: twice the CTAs for a small batch) or 128 (two CTAs per tile, 64 rows each).
// Schedules: unfused (the reference's order: cur GEMM -> gate -> res / skip GEMMs -> residual -> next layer) and FUSED (one
// MMA round trip per layer: a_l = (Lh + Bh'_l) + Wprev_l.x_l[t-d] + Wcur_l.x_{l-1} + Wf_l.h_{l-1} with Wf_l = Wcur_l.Wres_{l-1}
// and Bh'_l = Bh_l + Wcur_l.Bres_{l-1} folded at pack time, issued together with Wres_{l-1}.h_{l-1} and Wskip_{l-1}.h_{l-1}).
//
// Replaces nv_wavenet_persistent.cuh + matrix_math.cuh + softmax.cuh of the reference for T_data = half.
// Numerical contract (oracle/wavenet_oracle.c, WNO_PREC_FP16): weights, biases, embeddings, Lh and every GEMM input
// rounded to fp16; fp32 accumulation; residual stream, skip sum and softmax in fp32.
#include "wn_common.h"
#include "wn_layout.cuh"
#include "wn_math.cuh"
#include "wn_sm90.cuh"

namespace {

using namespace sm90;

constexpr int R = 64, A = 256;
constexpr int TILE = 16384;                 // [128 rows x 64 fp16] K-major SW128: one weight chunk / ring stage
constexpr int TU = 64;                      // utterances per CTA tile = rows of every activation tile = M of the MMA
constexpr int ATILE = TU * 128;             // [64 rows x 64 fp16] activation tile
constexpr int NCONS = 256;                  // two consumer warpgroups
constexpr int NT = NCONS + 32;              // + the TMA producer warp

struct TcImage {                            // byte offsets inside the packed image
    size_t layer_bytes, off_out, off_bias, total;
    size_t b_bh, b_bres, b_bskp, b_bzs, b_bza, b_bhf;     // float offsets inside the bias block
    size_t l_wf;                                   // byte offset of the folded matrix Wcur_l . Wres_{l-1} inside a layer block
};
__host__ __device__ inline TcImage tc_image(int S, int L)
{
    TcImage im;
    im.l_wf = (size_t)TILE * 2 + TILE / 2 + (size_t)(S / 128) * TILE;           // Wprev | Wcur | Wres | Wskip chunks | Wf
    im.layer_bytes = im.l_wf + TILE;
    im.off_out = (size_t)L * im.layer_bytes;
    im.off_bias = im.off_out + (size_t)(S / 64) * 2 * TILE + (size_t)(A / 64) * 2 * TILE;
    im.b_bh = 0;
    im.b_bres = im.b_bh + (size_t)L * 128;
    im.b_bskp = im.b_bres + (size_t)L * 64;
    im.b_bzs = im.b_bskp + (size_t)L * S;
    im.b_bza = im.b_bzs + A;
    im.b_bhf = im.b_bza + A;
    im.total = im.off_bias + (im.b_bhf + (size_t)L * 128) * sizeof(float);
    return im;
}

__host__ __device__ inline size_t tc_smem_bytes(int nstage)
{
    // alignment slack + weight ring + x and h tiles (two each) + 4 k-tiles of relu(skip) / relu(Zs) + fp32 logits + sampled indices + barriers
    return 1024 + (size_t)nstage * TILE + 4 * ATILE + 4 * ATILE + (size_t)TU * A * sizeof(float) + TU * sizeof(int) + 2 * (size_t)nstage * 8;
}

// Conditioning in the tensor-core layout: fp16 [N][L][Bpad rows][2 halves of 64 channels], tiled per c.tc_tile utterances;
// inside a tile: [half][row][128 B], 16-byte chunks XOR-swizzled with (row & 7) -- i.e. exactly the K-major
// SWIZZLE_128B image of an MMA A-operand tile, so a 1-D bulk TMA copy of rows*128 bytes needs no further shuffling.
__host__ __device__ inline int cond_rows(int B, int tile, int TU) { const int r = B - tile * TU; return r >= TU ? TU : ((r + 7) & ~7); }
__host__ __device__ inline size_t cond_bpad(int B, int TU) { const int nt = (B + TU - 1) / TU; return (size_t)(nt - 1) * TU + cond_rows(B, nt - 1, TU); }

// The tensor-core layouts for wn_layout.cuh: a unit is one 16-byte chunk of 8 channels in both.
struct TcLayout {
    using TD = __half;
    static constexpr int STORE_UNIT = 8, RING_UNIT = 8;
    // chunk k of the 2R channels of utterance b: half k / 8, chunk k mod 8 of its 128-byte row
    static __device__ WnVec<__half, 8>* store_unit(const WnConfig& c, void* store, size_t sl, int b, int k)
    {
        const int TU = c.tc_tile, tile = b / TU, r = b % TU, half = k >> 3, q = k & 7;
        return reinterpret_cast<WnVec<__half, 8>*>(static_cast<unsigned char*>(store) + (sl * cond_bpad(c.B, TU) + (size_t)tile * TU) * 256 +
                                                   (size_t)half * cond_rows(c.B, tile, TU) * 128 + (size_t)r * 128 + (size_t)((q ^ (r & 7)) << 4));
    }
    // The history ring: each entry (slot x L + layer) holds one 16 KB SW128 tile image per c.tc_tile utterances of the engine's
    // batch, row r = b mod tc_tile of a tile at bytes [128 r, 128 r + 128) in the channel order publish_x writes (its 16-byte chunks
    // permuted by r & 7).  Chunk q holds channels [8 q, 8 q + 8).
    static __device__ WnVec<__half, 8>* ring_unit(const WnConfig& c, void* ring, size_t e, int, int b, int q)
    {
        const int TU = c.tc_tile;
        return reinterpret_cast<WnVec<__half, 8>*>(static_cast<unsigned char*>(ring) + (e * ((c.B + TU - 1) / TU) + b / TU) * TILE +
                                                   sw128_offset(b % TU, 8 * q));
    }
    static size_t store_bytes(const WnConfig& c) { return (size_t)c.N * c.L * cond_bpad(c.B, c.tc_tile) * 256; }
    static size_t ring_bytes(const WnConfig& c)
    {
        const size_t tiled = (size_t)(c.maxDil + 1) * c.L * ((c.B + c.tc_tile - 1) / c.tc_tile) * TILE;
        const size_t plain = wn_stream_family.ring_bytes(c);
        return tiled > plain ? tiled : plain;
    }
};

// ------------------------------------------------------------------------------------------------ pack
// blob (fp16, column-major matrices as uploaded) -> tiled / swizzled weight image + fp32 bias block
__global__ void tc_pack_kernel(WnParams p, unsigned char* __restrict__ img, TcImage im)
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
    auto put = [&](size_t chunk_off, int row, int k, __half v) { *reinterpret_cast<__half*>(img + chunk_off + sw128_offset(row, k)) = v; };
    // per layer
    for (size_t i = g0; i < (size_t)L * 128 * 64; i += gstride) {
        const int l = (int)(i / (128 * 64)), c = (int)(i % (128 * 64)) / 64, k = (int)(i % 64);
        const size_t lb = (size_t)l * im.layer_bytes;
        put(lb, c, k, Wprev[(size_t)l * 128 * 64 + c + (size_t)k * 128]);
        put(lb + TILE, c, k, Wcur[(size_t)l * 128 * 64 + c + (size_t)k * 128]);
        if (c < 64) put(lb + 2 * TILE, c, k, Wres[(size_t)l * 64 * 64 + c + (size_t)k * 64]);
    }
    for (size_t i = g0; i < (size_t)L * S * 64; i += gstride) {
        const int l = (int)(i / ((size_t)S * 64)), s = (int)((i / 64) % S), k = (int)(i % 64);
        put((size_t)l * im.layer_bytes + 2 * TILE + TILE / 2 + (size_t)(s / 128) * TILE, s % 128, k, Wskip[(size_t)l * S * 64 + s + (size_t)k * S]);
    }
    // folded matrix of the fused schedule: Wf_l = Wcur_l . Wres_{l-1} (fp32 accumulation of the fp16 factors, one rounding),
    // so that Wcur_l . x_l = Wcur_l . x_{l-1} + Wf_l . h_{l-1} + Wcur_l . Bres_{l-1}
    for (size_t i = g0; i < (size_t)L * 128 * 64; i += gstride) {
        const int l = (int)(i / (128 * 64)), c = (int)(i % (128 * 64)) / 64, k = (int)(i % 64);
        if (l == 0) continue;
        float acc = 0.f;
        for (int j = 0; j < 64; j++)
            acc = fmaf(__half2float(Wcur[(size_t)l * 128 * 64 + c + (size_t)j * 128]), __half2float(Wres[(size_t)(l - 1) * 64 * 64 + j + (size_t)k * 64]), acc);
        put((size_t)l * im.layer_bytes + im.l_wf, c, k, __float2half_rn(acc));
    }
    // output layers: chunk (kt, nh) = rows a in [128 nh, +128), k in [64 kt, +64)
    for (size_t i = g0; i < (size_t)A * S; i += gstride) {
        const int a = (int)(i / S), s = (int)(i % S);
        put(im.off_out + (size_t)((s / 64) * 2 + a / 128) * TILE, a % 128, s % 64, Wzs[a + (size_t)s * A]);
    }
    const size_t off_wza = im.off_out + (size_t)(S / 64) * 2 * TILE;
    for (size_t i = g0; i < (size_t)A * A; i += gstride) {
        const int a = (int)(i / A), z = (int)(i % A);
        put(off_wza + (size_t)((z / 64) * 2 + a / 128) * TILE, a % 128, z % 64, Wza[a + (size_t)z * A]);
    }
    // biases -> fp32; running prefix of the skip biases (the skip sum is accumulated without biases)
    float* bias = reinterpret_cast<float*>(img + im.off_bias);
    const __half* Bh = static_cast<const __half*>(p.Bh);
    const __half* Bres = static_cast<const __half*>(p.Bres);
    const __half* Bskip = static_cast<const __half*>(p.Bskip);
    for (size_t i = g0; i < (size_t)L * 128; i += gstride) {
        const int l = (int)(i / 128), c = (int)(i % 128);
        const float bh = __half2float(Bh[i]);
        bias[im.b_bh + i] = bh;
        float acc = 0.f;                                        // Wcur_l . Bres_{l-1}
        if (l > 0)
            for (int j = 0; j < 64; j++)
                acc = fmaf(__half2float(Wcur[(size_t)l * 128 * 64 + c + (size_t)j * 128]), __half2float(Bres[(size_t)(l - 1) * 64 + j]), acc);
        bias[im.b_bhf + i] = bh + acc;
    }
    for (size_t i = g0; i < (size_t)L * 64; i += gstride) bias[im.b_bres + i] = __half2float(Bres[i]);
    for (size_t s = g0; s < (size_t)S; s += gstride) {
        float acc = 0.f;
        for (int l = 0; l < L; l++) { acc += __half2float(Bskip[(size_t)l * S + s]); bias[im.b_bskp + (size_t)l * S + s] = acc; }
    }
    for (size_t i = g0; i < (size_t)A; i += gstride) {
        bias[im.b_bzs + i] = __half2float(static_cast<const __half*>(p.Bzs)[i]);
        bias[im.b_bza + i] = __half2float(static_cast<const __half*>(p.Bza)[i]);
    }
}

// ------------------------------------------------------------------------------------------------ helpers
using wn::pack_h2;
using wn::unpack_h2;
// two consecutive fp16 (k even) of row `row` of a SW128 tile, in shared or global memory
__device__ __forceinline__ void st_pair(unsigned char* tile, int row, int k, float v0, float v1)
{
    *reinterpret_cast<uint32_t*>(tile + sw128_offset(row, k)) = pack_h2(v0, v1);
}
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// Accumulator fragment of a warpgroup (wn_sm90.cuh): thread i holds rows r0 = 16 (i / 32) + (i % 32) / 4 and r0 + 8, and in
// every 8-column group j the columns 8 j + 2 (i % 4) + {0, 1}.  Index 4 j + 2 r + e of a fragment array = row r0 + 8 r,
// column 8 j + 2 (i % 4) + e.  x, the gate inputs and Dx of one thread are the same 16 (row, channel) pairs.
// MODELS: p.group_model is set, and the CTA's weights are its tile's model's (a model group is one tile, DESIGN.md §6)
template <int S, bool FUSED, bool MODELS>
__global__ void __launch_bounds__(NT, 1) wn_tc_kernel(const WnParams p, const unsigned char* __restrict__ img0, const int nstage, const int tu)
{
    constexpr int SKN = S / 2;                     // skip columns per warpgroup
    constexpr int SKC = S / 128;                   // skip weight chunks per layer
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    // 1024-byte alignment by OFFSET (not by pointer round-trip through an integer): the compiler keeps knowing these
    // are shared-memory addresses and emits LDS/STS instead of generic LD/ST
    unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int L = p.L, B = p.B;
    const TcImage im = tc_image(S, L);

    unsigned char* ring = smem;                                    // nstage x 16 KB
    unsigned char* t_xb = ring + (size_t)nstage * TILE;            // x tiles [2]: A operand of Wcur (FUSED: by layer parity)
    unsigned char* t_hb = t_xb + 2 * ATILE;                        // h tiles [2]: A operand of Wres, Wskip (and Wf)
    unsigned char* t_big = t_hb + 2 * ATILE;                       // 4 k-tiles: relu(skip), then relu(Zs)
    float* s_z = reinterpret_cast<float*>(t_big + 4 * ATILE);      // [TU][A] logits, then exp(z - max)
    int* s_y = reinterpret_cast<int*>(s_z + TU * A);               // [TU] sampled index
    uint64_t* w_full = reinterpret_cast<uint64_t*>(s_y + TU);
    uint64_t* w_empty = w_full + nstage;

    const int tid = threadIdx.x;
    const int sub = tu > TU ? tu / TU : 1;                         // CTAs per tile
    const int tile = blockIdx.x / sub, ntiles = gridDim.x / sub;
    const WnGroupWeights gw = MODELS ? wn_group_weights(p, tile * tu) : WnGroupWeights{0, img0};
    const unsigned char* __restrict__ img = gw.image;
    const int row0 = (blockIdx.x % sub) * TU;                      // first row of this CTA inside its tile
    const int live = tu < TU ? tu : TU;                            // MMA rows that hold utterances
    const int slots = p.maxDil + 1;
    const int t_begin = p.init_sample, t_end = p.init_sample + p.count;
    // t below is a buffer position; the history goes by the utterance's time (DESIGN.md §6): x_l[t-d] exists iff t + t_hist >= d,
    // and position t has the ring slot (t + slot_shift) % slots (the sum is >= 0 for every t >= t_begin - maxDil)
    const int t_hist = p.hist_t - t_begin;
    const int slot_shift = p.ring_slot - t_begin % slots + slots;
    unsigned char* gring = static_cast<unsigned char*>(p.ring);
    auto ring_tile = [&](int t, int l) -> unsigned char* {
        return gring + (((size_t)((t + slot_shift) % slots) * L + l) * ntiles + tile) * (size_t)TILE + (size_t)row0 * 128;
    };
    // conditioning tile geometry (see TcLayout::store_unit): [2 halves][c_rows][128 B]; this CTA's rows of each half land in a ring
    // stage at offsets 0 and ATILE
    const int c_rows = cond_rows(B, tile, tu);
    const uint32_t c_bytes = (uint32_t)c_rows * 128u;
    const int c_here = min(max(c_rows - row0, 0), TU);
    const uint32_t c_bytes_here = (uint32_t)c_here * 128u;
    const size_t c_bpad = cond_bpad(B, tu);
    const unsigned char* gcond = static_cast<const unsigned char*>(p.Lh);
    auto cond_ptr = [&](int t, int l) -> const unsigned char* {
        return gcond + (((size_t)t * L + l) * c_bpad + (size_t)tile * tu) * 256 + (size_t)row0 * 128;
    };

    if (tid == 0) {
        for (int s = 0; s < nstage; s++) { mbar_init(&w_full[s], 1); mbar_init(&w_empty[s], NCONS); }
        fence_mbar_init();
    }
    __syncthreads();

    if (tid >= NCONS) {
        // =============================================================== TMA producer (one lane)
        // Chunk order = consumption order, per sample:
        //   unfused, per layer l:  Lh[t][l] | x_l[t-d] Wprev_l (if t >= d) | Wcur_l | Wres_l | Wskip_l (S/128 chunks)
        //   FUSED:   layer 0:      Lh[t][0] | x_0[t-1] Wprev_0 (if t >= 1) | Wcur_0
        //            layer l > 0:  Lh[t][l] | x_l[t-d] Wprev_l (if t >= d) | Wcur_l | Wf_l | Wres_{l-1} | Wskip_{l-1}
        //            then:         Wres_{L-1} | Wskip_{L-1}
        //   then the output layers, chunk (kt, nh) in the image's order.
        if (tid == NCONS) {
            int stage = 0;
            uint32_t ph = 1;
            auto put2 = [&](const void* src0, uint32_t bytes0, const void* src1, uint32_t bytes1) {
                mbar_wait(&w_empty[stage], ph);
                mbar_arrive_expect_tx(&w_full[stage], bytes0 + bytes1);
                if (bytes0) tma_load_1d(ring + (size_t)stage * TILE, src0, bytes0, &w_full[stage]);
                if (bytes1) tma_load_1d(ring + (size_t)stage * TILE + ATILE, src1, bytes1, &w_full[stage]);
                if (++stage == nstage) { stage = 0; ph ^= 1; }
            };
            auto put = [&](const void* src, uint32_t bytes) { put2(src, bytes, nullptr, 0); };
            auto res_skip = [&](int l) {
                const unsigned char* lw = img + (size_t)l * im.layer_bytes;
                put(lw + 2 * TILE, TILE / 2);
                for (int c = 0; c < SKC; c++) put(lw + 2 * TILE + TILE / 2 + (size_t)c * TILE, TILE);
            };
            for (int t = t_begin; t < t_end; t++) {
                int d = 1;                                              // dilation of layer l (nv_wavenet.cuh:99-111)
                for (int l = 0; l < L; l++) {
                    const unsigned char* lw = img + (size_t)l * im.layer_bytes;
                    put2(cond_ptr(t, l), c_bytes_here, cond_ptr(t, l) + c_bytes, c_bytes_here);
                    if (t + 1 < t_end && c_bytes_here) tma_prefetch_l2(cond_ptr(t + 1, l), c_bytes_here);
                    if (t + t_hist >= d) { put(ring_tile(t - d, l), ATILE); put(lw, TILE); }
                    put(lw + TILE, TILE);
                    if (FUSED) {
                        if (l > 0) { put(lw + im.l_wf, TILE); res_skip(l - 1); }
                    } else {
                        res_skip(l);
                    }
                    d <<= 1; if (d > p.maxDil) d = 1;
                }
                if (FUSED) res_skip(L - 1);
                for (int c = 0; c < (S / 64) * 2 + (A / 64) * 2; c++) put(img + im.off_out + (size_t)c * TILE, TILE);
            }
        }
        return;
    }

    // =============================================================== consumers: two warpgroups
    const int wg = tid >> 7, i = tid & 127;
    const int r0 = 16 * (i >> 5) + ((i & 31) >> 2), cq = 2 * (i & 3);
    const int ch0 = 32 * wg + cq;                  // residual / gate channel of fragment column 0
    int bb[2];
    bool valid[2];
    int yp[2], yc[2];
#pragma unroll
    for (int r = 0; r < 2; r++) {
        bb[r] = tile * tu + row0 + r0 + 8 * r;
        valid[r] = r0 + 8 * r < live && bb[r] < B;
        yp[r] = valid[r] ? p.yPrev[bb[r]] : 0;
        yc[r] = valid[r] ? p.yCur[bb[r]] : 0;
    }
    const __half* embPrev = gw.at<__half>(p.embPrev);
    const __half* embCur = gw.at<__half>(p.embCur);
    const float* gbias = reinterpret_cast<const float*>(img + im.off_bias);

    int stage = 0;
    uint32_t ph = 0;
    auto take = [&](int& s) -> const unsigned char* {              // next ring stage, once its data has landed
        s = stage;
        mbar_wait(&w_full[stage], ph);
        if (++stage == nstage) { stage = 0; ph ^= 1; }
        return ring + (size_t)s * TILE;
    };
    auto release = [&](int s) { mbar_arrive(&w_empty[s]); };
    auto desc = [](const void* p_) { return make_desc_sw128(smem_u32(p_)); };

    float x[16];                                   // residual stream (fp32) of this thread's 16 (row, channel) pairs
    float acc_s[SKN / 2];                          // skip sum over the layers, without biases
    float acc_x[16];                               // Dx = Wres.h of the latest residual GEMM

    for (int t = t_begin; t < t_end; t++) {
        const bool dump = p.dump && (t == t_end - 1);
        // ---------------- embedding: x0 = tanh(embPrev[yPrev] + embCur[yCur])   (reference.cpp:42-57)
#pragma unroll
        for (int r = 0; r < 2; r++)
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int c = ch0 + 8 * j;
                const float2 fa = __half22float2(*reinterpret_cast<const __half2*>(embPrev + (size_t)yp[r] * R + c));
                const float2 fc = __half22float2(*reinterpret_cast<const __half2*>(embCur + (size_t)yc[r] * R + c));
                float e0 = fa.x + fc.x, e1 = fa.y + fc.y;
                if (p.tanhEmbed) { e0 = wn::tanhf_fast(e0); e1 = wn::tanhf_fast(e1); }
                if (!valid[r]) { e0 = 0.f; e1 = 0.f; }
                x[4 * j + 2 * r] = e0; x[4 * j + 2 * r + 1] = e1;
            }
        // x tile and history ring: both hold x_l as the SW128 image of 64 rows (the ring is read back by TMA d samples later)
        auto publish_x = [&](unsigned char* xt, unsigned char* gdst) {
#pragma unroll
            for (int r = 0; r < 2; r++)
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    st_pair(xt, r0 + 8 * r, ch0 + 8 * j, x[4 * j + 2 * r], x[4 * j + 2 * r + 1]);
                    st_pair(gdst, r0 + 8 * r, ch0 + 8 * j, x[4 * j + 2 * r], x[4 * j + 2 * r + 1]);
                }
            fence_proxy_async_global();
        };
        publish_x(t_xb, ring_tile(t, 0));
        fence_proxy_async_smem();
        consumer_sync();                                                // x_0 tile complete

        // Wres_l.h -> acc_x and Wskip_l.h -> acc_s (issued into the current wgmma batch; the caller commits and waits)
        auto issue_res_skip = [&](int l, const unsigned char* th, int& sr, int (&sk)[SKC]) {
            const unsigned char* wr = take(sr);
            const unsigned char* wk[SKC];
#pragma unroll
            for (int c = 0; c < SKC; c++) wk[c] = take(sk[c]);
            const uint64_t dh = desc(th), dr = desc(wr + 32 * wg * 128);
            const uint64_t ds = (S == 256) ? desc(wk[wg]) : desc(wk[0] + SKN * wg * 128);
#pragma unroll
            for (int k = 0; k < 4; k++) {
                wgmma_f16<32>(acc_x, dh + 2 * k, dr + 2 * k, k > 0);
                wgmma_f16<SKN>(acc_s, dh + 2 * k, ds + 2 * k, l > 0 || k > 0);
            }
        };
        auto release_res_skip = [&](int sr, const int (&sk)[SKC]) {
            release(sr);
#pragma unroll
            for (int c = 0; c < SKC; c++) release(sk[c]);
        };
        // residual: x += Dx + Bres_l   (reference.cpp:82-84), then the dumps of layer l
        auto residual = [&](int l) {
#pragma unroll
            for (int r = 0; r < 2; r++)
#pragma unroll
                for (int j = 0; j < 4; j++)
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        const int q = 4 * j + 2 * r + e, c = ch0 + 8 * j + e;
                        x[q] = valid[r] ? x[q] + (acc_x[q] + gbias[im.b_bres + (size_t)l * 64 + c]) : 0.f;
                        if (dump && valid[r]) p.xtOut[((size_t)l * B + bb[r]) * R + c] = x[q];
                    }
            if (dump && l + 1 < L) {                                    // skip sum through layer l (the last one is dumped after relu)
#pragma unroll
                for (int j = 0; j < SKN / 8; j++)
#pragma unroll
                    for (int e = 0; e < 4; e++) {
                        const int r = e >> 1, s = SKN * wg + 8 * j + cq + (e & 1);
                        if (valid[r]) p.skipOut[((size_t)l * B + bb[r]) * S + s] = acc_s[4 * j + e] + gbias[im.b_bskp + (size_t)l * S + s];
                    }
            }
        };

        int d = 1;
        for (int l = 0; l < L; l++) {
            // ---------------- Lh[t][l] + Bh (FUSED, l > 0: Bh') of this thread's gate inputs, from the TMA-fed conditioning chunk
            float cnd_a[16], cnd_g[16];
            {
                int sc;
                const unsigned char* cb = take(sc);
                const float* bh = gbias + ((FUSED && l > 0) ? im.b_bhf : im.b_bh) + (size_t)l * 128;
#pragma unroll
                for (int r = 0; r < 2; r++)
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        const int c = ch0 + 8 * j, row = r0 + 8 * r;
                        const float2 la = unpack_h2(*reinterpret_cast<const uint32_t*>(cb + sw128_offset(row, c)));
                        const float2 lg = unpack_h2(*reinterpret_cast<const uint32_t*>(cb + ATILE + sw128_offset(row, c)));
                        const float2 ba = *reinterpret_cast<const float2*>(bh + c);
                        const float2 bg = *reinterpret_cast<const float2*>(bh + 64 + c);
                        cnd_a[4 * j + 2 * r] = la.x + ba.x; cnd_a[4 * j + 2 * r + 1] = la.y + ba.y;
                        cnd_g[4 * j + 2 * r] = lg.x + bg.x; cnd_g[4 * j + 2 * r + 1] = lg.y + bg.y;
                    }
                release(sc);
            }
            // ---------------- pre-activation: Wprev.x[t-d] + Wcur.x   (reference.cpp:67-80); FUSED: x = x_{l-1}, + Wf.h_{l-1}
            const unsigned char* t_x = t_xb + (FUSED ? (size_t)((l + 1) & 1) * ATILE : 0);     // FUSED, l > 0: x_{l-1}
            const unsigned char* t_hp = t_hb + (size_t)((l + 1) & 1) * ATILE;                  // FUSED: h_{l-1}
            float acc_a[16], acc_g[16];
            {
                const bool hp = t + t_hist >= d;
                int sh = 0, sp = 0, sw, sf = 0, sr = 0, sk[SKC];
                wgmma_fence();
                if (hp) {
                    const uint64_t dhx = desc(take(sh));
                    const unsigned char* wp = take(sp);
                    const uint64_t dpa = desc(wp + 32 * wg * 128), dpg = desc(wp + (64 + 32 * wg) * 128);
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        wgmma_f16<32>(acc_a, dhx + 2 * k, dpa + 2 * k, k > 0);
                        wgmma_f16<32>(acc_g, dhx + 2 * k, dpg + 2 * k, k > 0);
                    }
                    wgmma_commit();
                }
                const unsigned char* wc = take(sw);
                const uint64_t dx = desc(l == 0 ? t_xb : t_x), dca = desc(wc + 32 * wg * 128), dcg = desc(wc + (64 + 32 * wg) * 128);
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    wgmma_f16<32>(acc_a, dx + 2 * k, dca + 2 * k, hp || k > 0);
                    wgmma_f16<32>(acc_g, dx + 2 * k, dcg + 2 * k, hp || k > 0);
                }
                if (FUSED && l > 0) {
                    wgmma_commit();
                    const unsigned char* wf = take(sf);
                    const uint64_t dh = desc(t_hp), dfa = desc(wf + 32 * wg * 128), dfg = desc(wf + (64 + 32 * wg) * 128);
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        wgmma_f16<32>(acc_a, dh + 2 * k, dfa + 2 * k, 1u);
                        wgmma_f16<32>(acc_g, dh + 2 * k, dfg + 2 * k, 1u);
                    }
                    wgmma_commit();
                    // the history / Wprev stages go back to the producer before the residual and skip chunks are taken: a
                    // warpgroup never holds more than five ring stages at once
                    if (hp) { wgmma_wait<2>(); release(sh); release(sp); }
                    issue_res_skip(l - 1, t_hp, sr, sk);
                }
                wgmma_commit();
                wgmma_wait<0>();
                if (hp && !(FUSED && l > 0)) { release(sh); release(sp); }
                release(sw);
                if (FUSED && l > 0) { release(sf); release_res_skip(sr, sk); }
            }
            if (FUSED) {
                // x_l = x_{l-1} + Wres_{l-1}.h_{l-1} + Bres_{l-1} -> x tile of parity l (next layer's Wcur operand) + history ring;
                // the other warpgroup may still read the tiles of parity l-1, never those of parity l (one barrier per layer)
                if (l > 0) {
                    residual(l - 1);
                    publish_x(t_xb + (size_t)(l & 1) * ATILE, ring_tile(t, l));
                }
            }
            // ---------------- gate: h = tanh(a) * sigmoid(g) -> h tile
            unsigned char* t_h = t_hb + (FUSED ? (size_t)(l & 1) * ATILE : 0);
#pragma unroll
            for (int r = 0; r < 2; r++)
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int q = 4 * j + 2 * r;
                    float h0 = wn::tanhf_fast(acc_a[q] + cnd_a[q]) * wn::sigmoidf_fast(acc_g[q] + cnd_g[q]);
                    float h1 = wn::tanhf_fast(acc_a[q + 1] + cnd_a[q + 1]) * wn::sigmoidf_fast(acc_g[q + 1] + cnd_g[q + 1]);
                    if (!valid[r]) { h0 = 0.f; h1 = 0.f; }
                    st_pair(t_h, r0 + 8 * r, ch0 + 8 * j, h0, h1);
                }
            fence_proxy_async_smem();
            consumer_sync();                                            // h_l (FUSED: and x_l) tiles complete
            if (!FUSED) {
                // ---------------- Dx = Wres.h (this warpgroup's 32 channels), skip += Wskip.h (its S/2 columns)
                int sr, sk[SKC];
                wgmma_fence();
                issue_res_skip(l, t_h, sr, sk);
                wgmma_commit();
                wgmma_wait<0>();
                release_res_skip(sr, sk);
                residual(l);
                if (l + 1 < L) {
                    publish_x(t_xb, ring_tile(t, l + 1));
                    fence_proxy_async_smem();
                    consumer_sync();                                    // x_{l+1} tile complete
                }
            }
            d <<= 1; if (d > p.maxDil) d = 1;
        }
        if (FUSED) {                                                    // Wres_{L-1}, Wskip_{L-1} on h_{L-1}
            int sr, sk[SKC];
            wgmma_fence();
            issue_res_skip(L - 1, t_hb + (size_t)((L - 1) & 1) * ATILE, sr, sk);
            wgmma_commit();
            wgmma_wait<0>();
            release_res_skip(sr, sk);
            residual(L - 1);
        }

        // ---------------- relu(skip) -> A operand of the first output layer   (reference.cpp:88-90)
#pragma unroll
        for (int j = 0; j < SKN / 8; j++)
#pragma unroll
            for (int r = 0; r < 2; r++) {
                float v[2];
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const int s = SKN * wg + 8 * j + cq + e;
                    v[e] = valid[r] ? fmaxf(acc_s[4 * j + 2 * r + e] + gbias[im.b_bskp + (size_t)(L - 1) * S + s], 0.f) : 0.f;
                    if (dump && valid[r]) p.skipOut[((size_t)(L - 1) * B + bb[r]) * S + s] = v[e];
                }
                const int s = SKN * wg + 8 * j + cq;
                st_pair(t_big + (size_t)(s >> 6) * ATILE, r0 + 8 * r, s & 63, v[0], v[1]);
            }
        fence_proxy_async_smem();
        consumer_sync();

        // ---------------- output layers: warpgroup w computes columns [128 w, 128 w + 128) of Zs, then of Za
        float acc_z[64];
        auto out_gemm = [&](int KT) {
            for (int kt = 0; kt < KT; kt++) {
                int s0, s1;
                const unsigned char* w0 = take(s0);
                const unsigned char* w1 = take(s1);
                const uint64_t da = desc(t_big + (size_t)kt * ATILE), dw = desc(wg ? w1 : w0);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; k++) wgmma_f16<128>(acc_z, da + 2 * k, dw + 2 * k, kt > 0 || k > 0);
                wgmma_commit();
                wgmma_wait<0>();
                release(s0); release(s1);
            }
        };
        out_gemm(S / 64);
        consumer_sync();                                                // both warpgroups are done reading relu(skip)
        // Zs = relu(Wzs . skip + Bzs)   (reference.cpp:96-98)
#pragma unroll
        for (int j = 0; j < 16; j++)
#pragma unroll
            for (int r = 0; r < 2; r++) {
                float v[2];
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const int a = 128 * wg + 8 * j + cq + e;
                    v[e] = valid[r] ? fmaxf(acc_z[4 * j + 2 * r + e] + gbias[im.b_bzs + a], 0.f) : 0.f;
                    if (dump && valid[r]) p.Zs[(size_t)bb[r] * A + a] = v[e];
                }
                const int a = 128 * wg + 8 * j + cq;
                st_pair(t_big + (size_t)(a >> 6) * ATILE, r0 + 8 * r, a & 63, v[0], v[1]);
            }
        fence_proxy_async_smem();
        consumer_sync();
        out_gemm(A / 64);
        // Za = Wza . Zs + Bza   (reference.cpp:100-104) -> shared memory, one fp32 row per utterance
#pragma unroll
        for (int j = 0; j < 16; j++)
#pragma unroll
            for (int e = 0; e < 4; e++) {
                const int r = e >> 1, a = 128 * wg + 8 * j + cq + (e & 1);
                const float z = acc_z[4 * j + e] + gbias[im.b_bza + a];
                s_z[(r0 + 8 * r) * A + a] = z;
                if (dump && valid[r]) p.Za[(size_t)bb[r] * A + a] = z;
            }
        consumer_sync();

        // ---------------- softmax + categorical sample   (reference.cpp:106-121)
        // Four consecutive threads per utterance, 64 logits each; the parts meet through warp shuffles.
        {
            const int row = tid >> 2, part = tid & 3, lane = tid & 31;
            const int b = tile * tu + row0 + row;
            const bool v = row < live && b < B;
            float* zr = s_z + row * A + 64 * part;
            float mx = zr[0];
            for (int a = 1; a < 64; a++) mx = fmaxf(mx, zr[a]);
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            float ps = 0.f;
            for (int a = 0; a < 64; a++) {
                const float ev = wn::exp2f_fast((zr[a] - mx) * 1.4426950408889634f);
                zr[a] = ev;
                ps += ev;
            }
            float pp[4];
#pragma unroll
            for (int k = 0; k < 4; k++) pp[k] = __shfl_sync(0xffffffffu, ps, (lane & ~3) + k);
            float off = 0.f, total = 0.f;
#pragma unroll
            for (int k = 0; k < 4; k++) { if (k == part) off = total; total += pp[k]; }
            const float target = (v ? __ldg(p.sel + (size_t)t * B + b) : 0.5f) * total;
            // owner = the part whose running-sum interval holds the target; the first and last parts take what is outside
            const bool mine = (part == 0 || !(target < off)) && (target < off + ps || part == 3);
            if (mine) {
                int yy = part == 3 ? A - 1 : 64 * part + 63;
                float run = off;
                for (int a = 0; a < 64; a++) {
                    run += zr[a];
                    if (target < run) { yy = 64 * part + a; break; }
                }
                s_y[row] = yy;
                if (v) p.yOut[(size_t)b * p.N + t] = yy;
            }
            if (dump && v) {
                const float inv = 1.f / total;
                for (int a = 0; a < 64; a++) p.P[(size_t)b * A + 64 * part + a] = zr[a] * inv;
            }
        }
        consumer_sync();
#pragma unroll
        for (int r = 0; r < 2; r++)
            if (valid[r]) {
                const int y = s_y[r0 + 8 * r];
                yp[r] = yc[r];
                yc[r] = p.forced ? p.forced[(size_t)bb[r] * p.N + t] : y;
            }
    }
    if (wg == 0 && (i & 3) == 0) {
#pragma unroll
        for (int r = 0; r < 2; r++)
            if (valid[r]) { p.yPrev[bb[r]] = yp[r]; p.yCur[bb[r]] = yc[r]; }
    }
}

int pick_nstage()
{
    for (int n = 8; n >= 5; n--)                                // the fused schedule holds up to five stages at once
        if (tc_smem_bytes(n) <= 227 * 1024) return n;
    return 0;
}

size_t image_bytes(const WnConfig& c) { return tc_image(c.S, c.L).total; }

cudaError_t wn_tc_pack(void* image, const WnParams& p, cudaStream_t stream)
{
    const TcImage im = tc_image(p.S, p.L);
    cudaError_t e = cudaMemsetAsync(image, 0, im.total, stream);
    if (e != cudaSuccess) return e;
    tc_pack_kernel<<<264, 256, 0, stream>>>(p, static_cast<unsigned char*>(image), im);
    return cudaGetLastError();
}

cudaError_t wn_launch_tc(const WnConfig& c, const WnParams& p, const void* tc_image_, cudaStream_t stream, WnLaunchInfo* info)
{
    const int tu = c.tc_tile;
    const bool fused = c.tc_fused;
    const int nstage = pick_nstage();
    if (nstage < 5 || (tu != 32 && tu != 64 && tu != 128)) return cudaErrorInvalidValue;
    const size_t smem = tc_smem_bytes(nstage);
    const int grid = (p.B + tu - 1) / tu * (tu > TU ? tu / TU : 1);
    const unsigned char* im8 = static_cast<const unsigned char*>(tc_image_);
    cudaError_t e = cudaErrorInvalidValue;
#define WN_TC_LAUNCH(SV, FV, MV)                                                                                     \
    do {                                                                                                             \
        e = cudaFuncSetAttribute(wn_tc_kernel<SV, FV, MV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);  \
        if (e != cudaSuccess) return e;                                                                              \
        wn_tc_kernel<SV, FV, MV><<<grid, NT, smem, stream>>>(p, im8, nstage, tu);                                   \
    } while (0)
#define WN_TC_LAUNCH_M(SV, FV) do { if (p.group_model) WN_TC_LAUNCH(SV, FV, true); else WN_TC_LAUNCH(SV, FV, false); } while (0)
    if (p.S == 256) { if (fused) WN_TC_LAUNCH_M(256, true); else WN_TC_LAUNCH_M(256, false); }
    else { if (fused) WN_TC_LAUNCH_M(128, true); else WN_TC_LAUNCH_M(128, false); }
#undef WN_TC_LAUNCH_M
#undef WN_TC_LAUNCH
    if (info) { info->kernel = NVWN_KERNEL_TENSORCORE; info->grid = grid; info->block = NT; info->smem_bytes = (int)smem; info->batch_per_cta = tu < TU ? tu : TU; info->cluster = 1; }
    return cudaGetLastError();
}

}  // namespace

bool wn_tc_supported(int R_, int S, int A_, int, int)
{
    return R_ == R && A_ == A && (S == 128 || S == 256);
}

// a model group is one tile: every CTA of a tile of 128 runs its model
static int tc_group_rows(const WnConfig& c) { return c.tc_tile; }

// convert is convert_rows with every row: the whole-store and the per-row paths are one kernel
const WnFamily wn_tc_family = {TcLayout::store_bytes, TcLayout::ring_bytes, image_bytes, wn_convert<TcLayout>, wn_readback<TcLayout>,
                               wn_clear_rows<TcLayout>, wn_convert_rows<TcLayout>, wn_put_history<TcLayout>, wn_get_history<TcLayout>,
                               wn_put_history_rows<TcLayout>, wn_get_history_rows<TcLayout>, wn_clear_times<TcLayout>, wn_tc_pack,
                               wn_launch_tc, true, tc_group_rows};
