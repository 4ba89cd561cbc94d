// wn_engine.cu -- host side of the WaveNet inference engine + the handle C-ABI (include/nvwn_b200.h).
//
// Owns every device buffer, uploads / converts weights and inputs, picks the kernel and launches it.
// Re-design of the reference host class nvWavenetInfer<T_weight,T_data,R,S,A> (nv_wavenet.cuh:220-640):
//   * all weights live in ONE packed device blob (so a multi-GPU job broadcasts it with a single NCCL call);
//   * fp32 -> fp16 conversion runs on the device from a pinned/device staging area, asynchronously;
//   * every buffer frees itself (DevBuf); pointer kinds are detected with cudaPointerGetAttributes().type
//     (the reference's attributes.memoryType no longer compiles, nv_wavenet_conversions.cuh:41);
//   * yOut copies use cudaMemcpyDefault, so `samples` may be host or device memory.
#include "../../include/nvwn_b200.h"
#include "wn_common.h"

#include <limits.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <memory>
#include <string>
#include <utility>
#include <vector>

namespace {

thread_local std::string g_err;

int fail(int code, const std::string& msg)
{
    g_err = msg;
    return code;
}

#define CK(call)                                                                                             \
    do {                                                                                                     \
        cudaError_t _e = (call);                                                                             \
        if (_e != cudaSuccess)                                                                               \
            return fail((int)_e, std::string(cudaGetErrorString(_e)) + " at " __FILE__ ":" + std::to_string(__LINE__)); \
    } while (0)

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Absolute samples [first, first + count) of the engine's N-sample buffers used as rings (count <= N), as at most two pieces
// (position, offset, length): samples first + off .. first + off + len - 1 sit at positions pos .. pos + len - 1.  The same split
// as infer.split_at_wrap.
struct WrapPiece {
    int pos, off, len;
};
struct WrapPieces {
    WrapPiece piece[2];
    int n;
    const WrapPiece* begin() const { return piece; }
    const WrapPiece* end() const { return piece + n; }
};
WrapPieces split_at_wrap(long long first, int count, int N)
{
    const int pos = (int)(first % N), head = count < N - pos ? count : N - pos;
    return {{{pos, 0, head}, {0, head, count - head}}, (head > 0) + (head < count)};
}

bool is_device_ptr(const void* p)
{
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
}

// A device allocation that frees itself, and reads as the pointer it holds.  alloc() replaces the buffer only once the new
// allocation has succeeded: a failed grow leaves the old one in place.
struct CudaFree {
    void operator()(void* p) const { cudaFree(p); }
};
template <typename T>
struct DevBuf : std::unique_ptr<T, CudaFree> {
    size_t bytes = 0;                        // of the allocation held
    operator T*() const { return this->get(); }
    cudaError_t alloc(size_t n)
    {
        void* p = nullptr;
        const cudaError_t ce = cudaMalloc(&p, n);
        if (ce == cudaSuccess) {
            this->reset(static_cast<T*>(p));
            bytes = n;
        }
        return ce;
    }
    // At least n bytes.  A larger buffer replaces a smaller one after a device synchronise, so that no launch reads the old one any
    // more; the contents do not carry over.
    cudaError_t reserve(size_t n)
    {
        if (n <= bytes) return cudaSuccess;
        const cudaError_t ce = this->get() ? cudaDeviceSynchronize() : cudaSuccess;
        return ce != cudaSuccess ? ce : alloc(n);
    }
};

// A conditioning producer (DESIGN.md §6): a network of C channels, upsampling window K and stride; `scratch` of cond_scratch()'s
// layout, chunks of up to `rows` (row, sample) rows; row b's frames [C][T[b]] at frames + b * cap * C; the row list and WnCondSlot
// table of the last production (device); per row on the host, the frames of its utterance (0: none) and its absolute start.
// Live, both producers (nvwn_cond_producer_open_live, _open_live_slots) keep row b's frames in a ring [C][ring] at frames + b * ring * C
// (cap = ring), T[b] counting the frames pushed; per row whether a live utterance is attached (per-slot only), the first frame it was
// attached with (0 for the whole batch) and the end `done` of its furthest production, in its own samples.
struct CondProducer {
    int C = 0, K = 0, stride = 0, rows = 0;
    int ring = 0;                            // frames per row of a live sequence's ring; 0: frames loaded whole
    DevBuf<float> scratch;
    DevBuf<float> frames;
    int cap = 0;
    DevBuf<char> tables;                     // int [B] rows, then WnCondSlot [B] at cond_table_offset
    std::vector<int> T;
    std::vector<long long> start;
    std::vector<char> live;
    std::vector<int> first;
    std::vector<long long> done;
};

}  // namespace

struct nvwn_engine : WnConfig {
    int impl, tanhEmbed, device;
    size_t td;                               // sizeof(TD)
    const WnFamily* family;                  // the kernel family of `kernel`: the layouts of Lh, ring and image, and the launch

    // bytes of a packed weight blob (TD elements, models[m].blob), and the offsets in it
    size_t blob_bytes = 0;
    size_t o_embPrev, o_embCur, o_Wprev, o_Wcur, o_Wres, o_Wskip, o_Wzs, o_Wza, o_Bh, o_Bres, o_Bskip, o_Bzs, o_Bza;

    DevBuf<void> Lh;                         // TD [N][L][B][2R]
    DevBuf<float> sel;                       // [N][B]
    DevBuf<int> forced;                      // [B][N]
    bool use_forced = false;
    DevBuf<int> yPrev, yCur, yOut;
    DevBuf<void> ring;
    long long next_t = 0;                    // absolute time of the next sample to generate: where nvwn_run_stream must continue
    DevBuf<float> xtOut, skipOut, Zs, Za, P;

    DevBuf<float> stage;                     // device fp32 staging of host sources (feed); fp16 engines allocate it at creation
    size_t stage_elems = 0;

    // continuous batching (nvwn_restart_slots): per slot, the absolute sample its utterance started at and its selector key; the
    // slot indices and seeds of the last per-slot call
    DevBuf<long long> origin;                // [B]
    DevBuf<unsigned long long> seed;         // [B]
    DevBuf<int> slot_rows;                   // [B]
    DevBuf<unsigned long long> slot_seeds;   // [B]
    // a per-slot call since the last nvwn_reset_history: its rows (history, conditioning, selectors) sit at the engine's batch
    // stride, which the kernels read at the run's, so until the next reset a run must take the whole batch
    bool slot_rows_used = false;
    // the batch_size of the last nvwn_prime_from_score since the last nvwn_reset_history, 0 if none: the plain history ring was
    // written at that stride, so until the next reset a run must take that batch
    int prime_bs = 0;
    // per-slot primes (nvwn_prime_slots_from_score): the scoring rows of the last call (device, [B]); and whether a slot was primed
    // before sample maxDil since the last nvwn_reset_history.  Such a slot's history holds real values at times the kernels would
    // skip as "before the start" (t < d_l), so while this is set every launch reads the ring at every step (fill_params), and the
    // entries of the negative times were zeroed in every row.
    DevBuf<int> prime_rows;
    bool early_prime = false;
    // device staging of slot states in host memory (nvwn_save_slots, nvwn_load_slots), grown on demand
    DevBuf<char> state_stage;

    // The models (DESIGN.md §6): model 0 is the engine's own weights (the setters), models 1 .. NVWN_MAX_MODELS - 1 copies of source
    // engines' (nvwn_set_model).  A model's blob and the family's image, packed from it before the first launch after a change, are
    // allocated by nvwn_create for model 0 and when first set for the others, and never move: model_tab holds their bases for the
    // kernels (device [NVWN_MAX_MODELS]).  group_tab is the model of each group of group_rows rows (device [ceil(B / group_rows)]),
    // and group_host its host copy, empty until nvwn_set_group_models: then launches look the models up.
    struct Model {
        DevBuf<char> blob;
        DevBuf<void> image;
        bool repack = true;
        DevBuf<void> score_image;            // the scorer's image of the model, allocated and packed on the first scoring call that
        bool score_repack = true;            // runs the model after a change
    };
    std::vector<Model> models;
    DevBuf<WnModel> model_tab;
    DevBuf<int> group_tab;
    std::vector<int> group_host;
    int group_rows = 0;

    // the conditioning producers of the whole-batch calls (nvwn_cond_producer_load / _run / _run_stream) and of the per-slot calls
    // (nvwn_cond_producer_set_weights / _set_slots / _run_slots): each has its own weights, frames and scratch, so the two sets of
    // calls may be interleaved
    CondProducer cond_whole, cond_slots;

    // teacher-forced scoring (nvwn_score): chunk scratch, allocated on the first call (each model's image is in models)
    DevBuf<char> score_scratch;
    int score_T = 0;                         // time steps per chunk: SCORE_ROWS / B
    // the open scoring stream (nvwn_score_stream): the absolute sample its next call starts at, -1 if none is open, its batch_size,
    // and whether it is packed (nvwn_score_stream_packed); its state is the layer fronts, the codes and, packed, the local-time
    // carry in score_scratch
    long long score_next = -1;
    int score_bs = 0;
    bool score_packed = false;
    // scoring by model (nvwn_set_score_models): the model of every row (host, empty until the first table: all 0); score_tab its
    // device form, the rows by model then row (WnScoreSegs::order) followed by the table itself; score_segs the device copy of a
    // call's segments
    std::vector<int> score_models;
    DevBuf<int> score_tab;
    DevBuf<WnScoreSegs> score_segs;

    DevBuf<float> lut_f;                     // mu-law decode tables (nvwn_get_audio): A floats, then 2 x A int16 (wrap / saturate)
    DevBuf<unsigned long long> trace;        // debug timeline (nvwn_debug_trace)
    int trace_t = -1;

    WnLaunchInfo last{};
    unsigned long long launches = 0;
};

namespace {

// Hands n units of `unit` fp32 values at `src` (host or device) to convert(src_dev, first_unit, num_units).  A host source goes
// through the engine's device staging buffer, whole units at a time, and the call waits for those copies: the buffer and the
// source are free again on return.  On fp32 engines only the row conversions (`rows`) need that, and allocate the buffer on first
// need: the other conversions are copies that also read host memory.
template <typename Convert>
int feed(nvwn_engine* e, const float* src, size_t n, size_t unit, bool rows, cudaStream_t stream, Convert convert)
{
    if (n == 0) return 0;
    if ((e->dtype != NVWN_FP16 && !rows) || is_device_ptr(src)) {
        CK(convert(src, 0, n));
        return 0;
    }
    if (!e->stage) CK(e->stage.alloc(e->stage_elems * sizeof(float)));
    const size_t chunk = e->stage_elems / unit;                              // >= 1: stage_elems holds a sample of the whole batch
    for (size_t done = 0; done < n; done += chunk) {
        const size_t m = n - done < chunk ? n - done : chunk;
        CK(cudaMemcpyAsync(e->stage, src + done * unit, m * unit * sizeof(float), cudaMemcpyHostToDevice, stream));
        CK(convert(e->stage, done, m));
    }
    CK(cudaStreamSynchronize(stream));
    return 0;
}

// Host array -> device scratch, stream-ordered, through a snapshot in pageable memory: a pageable source is staged before
// cudaMemcpyAsync returns, so the caller's array (pinned or not) is free again on return.
template <typename T>
int copy_snapshot(void* dst_dev, const T* src, size_t n, cudaStream_t stream)
{
    const std::vector<T> snap(src, src + n);
    CK(cudaMemcpyAsync(dst_dev, snap.data(), n * sizeof(T), cudaMemcpyHostToDevice, stream));
    return 0;
}

// Where a producer's scratch holds each part, in floats from its start: Wu [C][C][K] | its [K][C][C] transpose WuT | bu [C] |
// Wc [L*2R][C] | bc [L*2R] | U chunk [rows][C] | output chunk [rows][L*2R], the last 16-byte aligned for the tiled projection's
// float4 stores
struct CondScratch {
    size_t wu, wut, bu, wc, bc, u, out, floats;
};
CondScratch cond_scratch(const nvwn_engine* e, int C, int K, int rows)
{
    const size_t lrow = (size_t)e->L * 2 * e->R, n_wu = (size_t)C * C * K;
    CondScratch o;
    o.wu = 0; o.wut = n_wu; o.bu = 2 * n_wu; o.wc = o.bu + C; o.bc = o.wc + lrow * C; o.u = o.bc + lrow;
    o.out = align_up(o.u + (size_t)rows * C, 4);
    o.floats = o.out + (size_t)rows * lrow;
    return o;
}

// bytes before the WnCondSlot table in a producer's `tables`
size_t cond_table_offset(const nvwn_engine* e) { return align_up((size_t)e->B * sizeof(int), 16); }

// Gives P the conditioning network, from host or device sources, and the transpose the kernels read; sizes its chunks to about
// 64 MB of fp32 and at least one sample of every row, and grows its scratch when that is too small.  Stream-ordered on `st`: the
// caller synchronises before the sources may be released.
int put_cond_network(nvwn_engine* e, CondProducer& P, const std::string& who, int C, int K, int stride, const float* Wu, const float* bu,
                     const float* Wc, const float* bc, cudaStream_t st)
{
    const size_t lrow = (size_t)e->L * 2 * e->R;                             // floats of one (row, sample) of conditioning
    const size_t rows = ((size_t)16 << 20) / lrow > (size_t)e->B ? ((size_t)16 << 20) / lrow : (size_t)e->B;
    const CondScratch o = cond_scratch(e, C, K, (int)rows);
    CK(P.scratch.reserve(o.floats * sizeof(float)));
    if (!P.tables) CK(P.tables.alloc(cond_table_offset(e) + (size_t)e->B * sizeof(WnCondSlot)));
    P.C = C; P.K = K; P.stride = stride; P.rows = (int)rows;
    float* w = P.scratch;
    cudaError_t ce = cudaSuccess;
    auto put = [&](size_t dst, const float* src, size_t n) { if (ce == cudaSuccess) ce = cudaMemcpyAsync(w + dst, src, n * sizeof(float), cudaMemcpyDefault, st); };
    put(o.wu, Wu, o.wut - o.wu); put(o.bu, bu, C); put(o.wc, Wc, o.bc - o.wc); put(o.bc, bc, lrow);
    if (ce == cudaSuccess) ce = wn_cond_transpose_wu(w + o.wut, w + o.wu, C, K, st);
    if (ce != cudaSuccess) return fail((int)ce, who + ": " + cudaGetErrorString(ce));
    return 0;
}

// Conditioning of absolute samples t_first .. t_first + count - 1 for rows rows[0..n) of P (host list; NULL: rows 0 .. B - 1 of
// the whole-batch producer, n = B), each read from its own utterance, into store positions pos .. pos + count - 1: the caller has
// checked the ranges, split them at the ring's wrap and put the rows' WnCondSlot table (and list) into P.tables.  Chunks of
// P.rows / n whole samples, stored by convert_rows, or for a whole batch by the family's convert: the latency family's convert
// writes 16-byte stores and zeroes the padding rows of the last tile, which convert_rows does not.
int produce(nvwn_engine* e, const CondProducer& P, const std::string& who, const int* rows, int n, long long t_first, int pos, int count,
            cudaStream_t st)
{
    const CondScratch o = cond_scratch(e, P.C, P.K, P.rows);
    float* w = P.scratch;
    const int* rows_dev = rows ? reinterpret_cast<const int*>(P.tables.get()) : nullptr;
    const WnCondSlot* tab = reinterpret_cast<const WnCondSlot*>(P.tables + cond_table_offset(e));
    long long end = LLONG_MAX;                                                // the earliest end of a listed utterance
    for (int i = 0; i < n; i++) {
        const int r = rows ? rows[i] : i;
        const long long end_r = P.start[r] + (long long)P.T[r] * P.stride;
        if (end_r < end) end = end_r;
    }
    const int chunk = P.rows / n;                                             // >= 1 as P.rows >= B
    cudaError_t ce = cudaSuccess;
    for (int done = 0; done < count && ce == cudaSuccess; done += chunk) {
        const int m = count - done < chunk ? count - done : chunk;
        const long long t0 = t_first + done;
        ce = wn_cond_produce_slots(w + o.out, w + o.u, P.frames, tab, w + o.wut, w + o.bu, w + o.wc, w + o.bc, n, P.C, P.K, P.stride, e->L, e->R,
                                   t0, m, end < t0 + m, P.ring > 0, st);
        if (ce == cudaSuccess)
            ce = rows ? e->family->convert_rows(*e, e->Lh, w + o.out, rows_dev, n, pos + done, m, st) : e->family->convert(*e, e->Lh, w + o.out, pos + done, m, st);
    }
    if (ce != cudaSuccess) return fail((int)ce, who + ": " + cudaGetErrorString(ce));
    return 0;
}

// The window of a call on absolute samples [first_sample, first_sample + count) of the engine's N-sample buffers used as rings:
// first_sample >= 0 and least <= count <= N.
int check_window(const nvwn_engine* e, const std::string& who, long long first_sample, int count, const char* count_name, int least)
{
    if (first_sample >= 0 && count >= least && count <= e->N) return 0;
    const std::string got = first_sample < 0 ? "first_sample " + std::to_string(first_sample) + " < 0" : std::string(count_name) + " = " + std::to_string(count);
    return fail(NVWN_EINVAL, who + ": need first_sample >= 0 and " + std::to_string(least) + " <= " + count_name + " <= num_samples (" +
                                 std::to_string(e->N) + ") of the engine; got " + got);
}

// The first frame that sample n of a sequence reads: frames ceil((n - K + 1) / stride) .. floor(n / stride), none below 0
long long first_frame(long long n, int K, int stride)
{
    const long long lo = n - K + 1;
    return lo <= 0 ? 0 : (lo + stride - 1) / stride;
}

// The batch a run, or a prime, may take: the tensor-core kernels take whole batches only, and so does every run after a per-slot
// call until nvwn_reset_history (slot_rows_used).
int check_run_batch(const nvwn_engine* e, const std::string& who, int batch)
{
    if (e->family->whole_batch && batch != e->B)
        return fail(NVWN_EINVAL, who + ": the tensor-core path needs batch_size equal to the engine's batch size (" + std::to_string(e->B) + "); got " +
                                     std::to_string(batch));
    if (e->slot_rows_used && batch != e->B)
        return fail(NVWN_EINVAL, who + ": after a per-slot call (nvwn_restart_slots, nvwn_set_conditioning_slots and the other *_slots calls) runs need "
                                     "batch_size equal to the engine's batch size (" + std::to_string(e->B) + ") until nvwn_reset_history; got " +
                                     std::to_string(batch));
    return 0;
}

// Checks a list of n indices (host memory): every one in [0, bound), none twice.  A refusal names an index as `noun` and follows the
// bound with `note`.
int check_list(const std::string& who, const int* list, int n, int bound, const char* noun, const char* note)
{
    std::vector<char> seen(bound, 0);
    for (int i = 0; i < n; i++) {
        const std::string x = std::string(noun) + " " + std::to_string(list[i]);
        if (list[i] < 0 || list[i] >= bound) return fail(NVWN_EINVAL, who + ": " + x + " is outside [0, " + std::to_string(bound) + ")" + note);
        if (seen[list[i]]) return fail(NVWN_EINVAL, who + ": " + x + " is given twice");
        seen[list[i]] = 1;
    }
    return 0;
}

// Checks the slot list of a per-slot call (host memory): 1 <= n <= B, every slot in [0, B), none twice.
int check_slots(const nvwn_engine* e, const std::string& who, const int* slots, int n)
{
    if (!slots) return fail(NVWN_EINVAL, who + ": slots is NULL");
    if (n < 1 || n > e->B) return fail(NVWN_EINVAL, who + ": need 1 <= n <= B (" + std::to_string(e->B) + "); got n = " + std::to_string(n));
    return check_list(who, slots, n, e->B, "slot", "");
}

// Checks a list of n scoring rows of the open scoring stream (host memory): every row in [0, Bs), none twice.
int check_rows(const nvwn_engine* e, const std::string& who, const int* rows, int n)
{
    return check_list(who, rows, n, e->score_bs, "row", " (the scoring stream's batch_size)");
}

// Checks that a model table names only model 0 and models given to nvwn_set_model: entry i of `what` ("group", "row") is models[i].
int check_models(const nvwn_engine* e, const std::string& who, const char* what, const int* models, int n)
{
    for (int i = 0; i < n; i++)
        if (models[i] < 0 || models[i] >= NVWN_MAX_MODELS || !e->models[models[i]].blob)
            return fail(NVWN_EINVAL, who + ": " + what + " " + std::to_string(i) + " names model " + std::to_string(models[i]) + ", which was never set");
    return 0;
}

// check_slots, then copies the list to slot_rows and the seeds, if any, to slot_seeds (device, stream-ordered), and marks the
// engine's rows as laid out for runs of the whole batch.  *seeds_dev: slot_seeds, or NULL without seeds (every seed 0).
int take_slots(nvwn_engine* e, const std::string& who, const int* slots, int n, const unsigned long long* seeds,
               const unsigned long long** seeds_dev, cudaStream_t stream)
{
    int rc = check_slots(e, who, slots, n);
    if (rc != 0) return rc;
    e->slot_rows_used = true;
    if ((rc = copy_snapshot(e->slot_rows, slots, n, stream))) return rc;
    if (seeds && (rc = copy_snapshot(e->slot_seeds, seeds, n, stream))) return rc;
    if (seeds_dev) *seeds_dev = seeds ? e->slot_seeds.get() : nullptr;
    return 0;
}

// Model m's weights changed: both its images are repacked before their next use.
void model_changed(nvwn_engine* e, int m) { e->models[m].repack = e->models[m].score_repack = true; }

// Model 0's weights changed: model_changed, and an open scoring stream ends (its carried layer inputs used the old weights).
void weights_changed(nvwn_engine* e)
{
    model_changed(e, 0);
    e->score_next = -1;
}

// Gives model m a blob and the family's image, and writes their bases into entry m of model_tab
int add_model(nvwn_engine* e, int m)
{
    nvwn_engine::Model fresh;
    CK(fresh.blob.alloc(e->blob_bytes));
    if (e->family->pack) CK(fresh.image.alloc(e->family->image_bytes(*e)));
    const WnModel bases{fresh.blob, fresh.image};
    CK(cudaMemcpy(e->model_tab + m, &bases, sizeof bases, cudaMemcpyHostToDevice));
    e->models[m] = std::move(fresh);
    return 0;
}

// Model 0's blob at byte offset off (TD, device) <- src (fp32, host or device), n elements
int upload(nvwn_engine* e, size_t off, const float* src, size_t n)
{
    void* dst = e->models[0].blob + off;
    return feed(e, src, n, 1, false, 0, [&](const float* s, size_t first, size_t m) {
        return e->dtype == NVWN_FP16 ? wn_f32_to_f16(static_cast<__half*>(dst) + first, s, m, 0)
                                     : cudaMemcpyAsync(static_cast<float*>(dst) + first, s, m * sizeof(float), cudaMemcpyDefault, 0);
    });
}

// dst (fp32, host or device) <- src (fp32 device)
int download(float* dst, const float* src, size_t n)
{
    CK(cudaMemcpy(dst, src, n * sizeof(float), cudaMemcpyDefault));
    return 0;
}

// The engine's kernel family and its variant, from its sizes, `impl` (an NVWN_KERNEL_* id forces a family) and the environment
// switches of INTEGRATION.md §1.  The only place the library reads the environment, once per engine: the conditioning store, the
// history ring and the weight image are laid out for what it decides.
void resolve_config(WnConfig& c, int impl)
{
    auto num = [](const char* name, int unset) { const char* v = getenv(name); return v ? atoi(v) : unset; };
    const int tc = wn_tc_supported(c.R, c.S, c.A, c.L, c.B) ? NVWN_KERNEL_TENSORCORE : NVWN_KERNEL_STREAM;
    const int lat = wn_lat_supported(c.R, c.S, c.A, c.L) ? NVWN_KERNEL_LATENCY : NVWN_KERNEL_STREAM;
    const char* fp16 = getenv("NVWN_FP16_KERNEL");
    if (c.dtype != NVWN_FP16 || impl == NVWN_KERNEL_STREAM) c.kernel = NVWN_KERNEL_STREAM;
    else if (impl == NVWN_KERNEL_TENSORCORE) c.kernel = tc;
    else if (impl == NVWN_KERNEL_LATENCY) c.kernel = lat;
    else if (fp16 && !strcmp(fp16, "stream")) c.kernel = NVWN_KERNEL_STREAM;
    else if (fp16 && !strcmp(fp16, "tc")) c.kernel = tc;
    else if (fp16 && !strcmp(fp16, "lat")) c.kernel = lat;
    // the latency kernels beat the tensor-core kernel even when their 16-utterance tiles need several waves (H100 80GB HBM3,
    // 400 W power limit, 2 560 utterances: 41.6 M against 14.1 M samples/s); NVWN_LAT_MAX_B caps the batch they take
    else c.kernel = lat == NVWN_KERNEL_LATENCY && c.B <= num("NVWN_LAT_MAX_B", INT_MAX) ? lat : tc;

    // tensor-core: 64-utterance tiles unless NVWN_TC_TILE (32 | 64 | 128) or NVWN_TC_NODUP (128) asks for another shape; the
    // unfused schedule unless NVWN_TC_FUSED is set and not "0", or the tiles are 32 utterances
    c.tc_tile = 64;
    c.tc_fused = false;
    if (c.kernel == NVWN_KERNEL_TENSORCORE) {
        const int t = num("NVWN_TC_TILE", 64);
        if (t == 32 || t == 128) c.tc_tile = t;
        if (getenv("NVWN_TC_NODUP")) c.tc_tile = 128;
        const char* fused = getenv("NVWN_TC_FUSED");
        c.tc_fused = (fused && fused[0] != '0') || c.tc_tile == 32;
    }
    c.lat_cluster = num("NVWN_LAT_CLUSTER", 1) != 0;
    const int bt = num("NVWN_STREAM_BT", 0);
    c.stream_bt = bt == 1 || bt == 2 || bt == 4 ? bt : 0;
    c.stream_ring = num("NVWN_STREAM_RING", 1) != 0;
}

// p's model pointers: the model whose blob starts at `blob`
void point_weights(const nvwn_engine* e, WnParams& p, const char* blob)
{
    p.embPrev = blob + e->o_embPrev; p.embCur = blob + e->o_embCur;
    p.Wprev = blob + e->o_Wprev; p.Wcur = blob + e->o_Wcur; p.Wres = blob + e->o_Wres; p.Wskip = blob + e->o_Wskip;
    p.Wzs = blob + e->o_Wzs; p.Wza = blob + e->o_Wza;
    p.Bh = blob + e->o_Bh; p.Bres = blob + e->o_Bres; p.Bskip = blob + e->o_Bskip; p.Bzs = blob + e->o_Bzs; p.Bza = blob + e->o_Bza;
}

// init_sample: buffer position of the first step; t_abs: its absolute time in the utterance batch (equal outside streaming use)
void fill_params(const nvwn_engine* e, WnParams& p, int init_sample, long long t_abs, int count, int num_samples, int batch, int dump)
{
    memset(&p, 0, sizeof p);
    p.L = e->L; p.R = e->R; p.S = e->S; p.A = e->A; p.maxDil = e->maxDil;
    p.B = batch; p.N = num_samples; p.init_sample = init_sample; p.count = count;
    p.ring_slot = (int)(t_abs % (e->maxDil + 1));
    p.hist_t = (int)(t_abs < e->maxDil && !e->early_prime ? t_abs : e->maxDil);
    p.tanhEmbed = e->tanhEmbed; p.dump = dump;
    point_weights(e, p, e->models[0].blob);
    p.Lh = e->Lh; p.sel = e->sel; p.forced = e->use_forced ? e->forced.get() : nullptr;
    p.yPrev = e->yPrev; p.yCur = e->yCur; p.ring = e->ring; p.yOut = e->yOut;
    p.xtOut = e->xtOut; p.skipOut = e->skipOut; p.Zs = e->Zs; p.Za = e->Za; p.P = e->P;
    p.trace = e->trace; p.trace_t = e->trace_t;
    p.group_rows = e->group_rows;
    if (!e->group_host.empty()) { p.group_model = e->group_tab; p.models = e->model_tab; }
}

// One generation launch: `count` steps from buffer position `pos` (pos + count <= num_samples, the yOut row stride), the first at
// absolute time t_abs.  Moves the engine's next sample to the end of the range.
int launch_steps(nvwn_engine* e, const char* who, int pos, long long t_abs, int count, int num_samples, int batch, int dump, cudaStream_t stream)
{
    WnParams p;
    fill_params(e, p, pos, t_abs, count, num_samples, batch, dump);
    if (count > 0) {
        const int rc = check_run_batch(e, who, batch);
        if (rc != 0) return rc;
        if (e->prime_bs && batch != e->prime_bs)
            return fail(NVWN_EINVAL, std::string(who) + ": after nvwn_prime_from_score runs need batch_size equal to the primed batch_size (" +
                                     std::to_string(e->prime_bs) + ") until nvwn_reset_history; got " + std::to_string(batch));
        for (nvwn_engine::Model& m : e->models) {
            if (!e->family->pack || !m.blob || !m.repack) continue;
            WnParams q = p;
            point_weights(e, q, m.blob);
            CK(e->family->pack(m.image, q, stream));
            m.repack = false;
        }
        CK(e->family->launch(*e, p, e->models[0].image, stream, &e->last));
        e->launches++;
    }
    e->next_t = t_abs + count;
    return 0;
}

// rows (t, b) of one scoring chunk; bounds the chunk scratch: DESIGN.md §5.4
constexpr int SCORE_ROWS = 16384;

// byte offsets of the scoring scratch, for the engine's B and N and a chunk of T steps
struct ScoreScratch {
    size_t audio, logp, bad, codes, starts, tau, carry, lh, xh, xf, H, lgt, bytes;
};
ScoreScratch score_scratch_layout(const nvwn_engine* e, int T)
{
    ScoreScratch o;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t r = off; off = align_up(off + bytes, 256); return r; };
    const size_t B = e->B, N = e->N, L = e->L, R = e->R, Tz = T;
    o.audio = take(B * N * sizeof(int));
    o.logp = take(B * N * sizeof(float));
    o.bad = take(sizeof(unsigned long long));
    o.codes = take(B * 2 * sizeof(int));
    o.starts = take(B * N);                  // packed scoring: the call's start flags, its chunk's local times and their carry
    o.tau = take(Tz * B * sizeof(int));
    o.carry = take(B * sizeof(int));
    o.lh = take(Tz * L * B * 2 * R * sizeof(float));
    o.xh = take(wn_score_xh_offset(e->L, e->L, e->maxDil, T, e->B, e->R) * sizeof(__half));
    o.xf = take(Tz * B * R * sizeof(float));
    o.H = take(Tz * B * L * R * sizeof(__half));
    o.lgt = take(Tz * B * e->A * sizeof(float));
    o.bytes = off;
    return o;
}

// The preamble of the calls that take the layer fronts of the open scoring stream (the primes, nvwn_score_save_states): an fp16
// engine with an open scoring stream of P >= 1 samples, not packed.  `fronts` says what the caller takes the fronts for.
int check_open_stream(const nvwn_engine* e, const std::string& who, const char* fronts)
{
    if (!e) return fail(NVWN_EINVAL, who + ": NULL engine");
    if (e->dtype != NVWN_FP16) return fail(NVWN_EUNSUPPORTED, who + ": only NVWN_FP16 engines can score");
    if (e->score_next < 1)
        return fail(NVWN_EINVAL, who + ": no open scoring stream (nvwn_score and weight changes end one): score the prompt with nvwn_score_stream "
                                       "from first_sample = 0 first");
    if (e->score_packed)
        return fail(NVWN_EUNSUPPORTED, who + ": the scoring stream is packed (nvwn_score_stream_packed): a row's layer fronts may hold an earlier "
                                             "utterance's inputs, so they are no " + fronts);
    return 0;
}

// The model scoring row b runs (nvwn_set_score_models)
int score_model(const nvwn_engine* e, int b) { return e->score_models.empty() ? 0 : e->score_models[b]; }

// A prime may only write a row or slot whose group generates with the model its scoring row was scored with: scoring rows
// rows[0..n) into slots slots[0..n) (NULL: 0 .. n - 1 for either)
int check_prime_model(const nvwn_engine* e, const std::string& who, const int* rows, const int* slots, int n)
{
    for (int i = 0; i < n; i++) {
        const int r = rows ? rows[i] : i, s = slots ? slots[i] : i;
        const int sm = score_model(e, r), gm = e->group_host.empty() ? 0 : e->group_host[s / e->group_rows];
        if (sm != gm)
            return fail(NVWN_EINVAL, who + ": row " + std::to_string(s) + " is in a group that runs model " + std::to_string(gm) + ", and its scoring row " +
                                           std::to_string(r) + " was scored with model " + std::to_string(sm) + ": set the scoring table (nvwn_set_score_models) "
                                           "to the group's model, or score the prompt on an engine holding that model and load its state (nvwn_score_save_states, "
                                           "nvwn_load_slots)");
    }
    return 0;
}

// Hands every layer's front of the open scoring stream of P samples to write(layer, src, tau, n): x_l of stream times [tau, P),
// tau = max(0, P - d_l), as fp16 [n][Bs][R] in the scoring scratch.  These are the entries a generation from stream time P reads
// (x_l[t - d_l] with t >= P); earlier times are never read (hist_t).
template <typename Write>
int put_fronts(const nvwn_engine* e, Write write)
{
    const long long P = e->score_next;
    const __half* xh = reinterpret_cast<const __half*>(e->score_scratch + score_scratch_layout(e, e->score_T).xh);
    for (int l = 0; l < e->L; l++) {
        const int d = wn_score_dilation(l, e->maxDil);
        const long long tau = P - d > 0 ? P - d : 0;
        CK(write(l, xh + wn_score_xh_offset(l, e->L, e->maxDil, e->score_T, e->B, e->R) + (size_t)(tau - (P - d)) * e->score_bs * e->R, tau,
                 (int)(P - tau)));
    }
    return 0;
}

// The sizes of a conditioning network: C >= 1 channels, window K >= stride >= 1
int check_cond_sizes(const std::string& who, int C, int K, int stride)
{
    if (C >= 1 && stride >= 1 && K >= stride) return 0;
    return fail(NVWN_EINVAL, who + ": bad sizes (need n_cond_channels >= 1 and window >= stride >= 1)");
}

// A live ring holds at least the frames one sample reads, and one frame more
int check_ring_frames(const std::string& who, int ring_frames, int K, int stride)
{
    const int least = (K + stride - 1) / stride + 1;
    if (ring_frames >= least) return 0;
    return fail(NVWN_EINVAL, who + ": ring_frames = " + std::to_string(ring_frames) + "; need at least ceil(window / stride) + 1 = " +
                                 std::to_string(least));
}

// Row r's entry of P's WnCondSlot table, with T frames
WnCondSlot cond_row(const CondProducer& P, int r, int T) { return {(long long)r * P.cap * P.C, P.start[r], T, P.ring}; }

// The WnCondSlot table of rows rows[0..n) (NULL: 0 .. n - 1) with their frames of now, and the row list if given, into P.tables in
// one copy staged from pageable memory in stream order: the caller's arrays are free again on return
int put_cond_table(const nvwn_engine* e, const CondProducer& P, const int* rows, int n, cudaStream_t st)
{
    const size_t off = cond_table_offset(e), skip = rows ? 0 : off;
    std::vector<char> host(off + (size_t)n * sizeof(WnCondSlot));
    if (rows) memcpy(host.data(), rows, (size_t)n * sizeof(int));
    WnCondSlot* tab = reinterpret_cast<WnCondSlot*>(host.data() + off);
    for (int i = 0; i < n; i++) tab[i] = cond_row(P, rows ? rows[i] : i, P.T[rows ? rows[i] : i]);
    CK(cudaMemcpyAsync(P.tables + skip, host.data() + skip, host.size() - skip, cudaMemcpyHostToDevice, st));
    return 0;
}

// A production of row r of a live sequence from sample n of its utterance reads frames from first_frame(n) on: they must still be in
// the ring, which holds [T - ring, T) and none before the frame the row was attached with.  `of` names the row's utterance in a refusal.
int check_held(const CondProducer& P, const std::string& who, int r, long long n, const std::string& of)
{
    const long long need = first_frame(n, P.K, P.stride), wrap = (long long)P.T[r] - P.ring, held = wrap > P.first[r] ? wrap : P.first[r];
    if (need >= held) return 0;
    return fail(NVWN_EINVAL, who + ": frame " + std::to_string(need) + ", which sample " + std::to_string(n) + of + " reads, has left the ring (it holds frames " +
                                 std::to_string(held) + " .. " + std::to_string(P.T[r] - 1) + ")");
}

// A push of num frames to row r of a live sequence overwrites frames [T - ring, T + num - ring): the samples from done[r] on read
// frames from first_frame(done[r]), and the frames before first[r] are gone already.  `of` names the row in a refusal.
int check_push(const CondProducer& P, const std::string& who, int r, int num, const std::string& of)
{
    const long long ff = first_frame(P.done[r], P.K, P.stride), keep = ff > P.first[r] ? ff : P.first[r];
    if ((long long)P.T[r] + num - P.ring <= keep) return 0;
    return fail(NVWN_EINVAL, who + ": " + std::to_string(num) + " frames would overwrite frame " + std::to_string(keep) + of + ", which sample " +
                                 std::to_string(P.done[r]) + " (not produced yet) reads; at most " + std::to_string(keep + P.ring - P.T[r]) +
                                 " frames fit before production moves on");
}

// Rows rows[0..n) of P (NULL: 0 .. n - 1) have been produced up to absolute sample `end`
void mark_produced(CondProducer& P, const int* rows, int n, long long end)
{
    for (int i = 0; i < n; i++) {
        const int r = rows ? rows[i] : i;
        if (end - P.start[r] > P.done[r]) P.done[r] = end - P.start[r];
    }
}

// Frames [rows][C][num] at src (host or device) -> frames T .. T + num - 1 of the rings of rows row .. row + rows - 1, split at the
// wrap.  A host source is snapshotted into pageable memory, which the copies stage before they return: the caller's array is free.
int put_live_frames(CondProducer& P, int row, int rows, long long T, const float* src, int num, cudaStream_t st)
{
    std::vector<float> snap;
    if (!is_device_ptr(src)) {
        snap.assign(src, src + (size_t)rows * P.C * num);
        src = snap.data();
    }
    const size_t f = sizeof(float);
    for (const WrapPiece& w : split_at_wrap(T, num, P.ring))
        CK(cudaMemcpy2DAsync(P.frames + (size_t)row * P.ring * P.C + w.pos, (size_t)P.ring * f, src + w.off, (size_t)num * f, (size_t)w.len * f,
                             (size_t)rows * P.C, cudaMemcpyDefault, st));
    return 0;
}

// Hands each layer's part of a slot state to part(layer, its byte offset in the state, d_l): [d_l][R] elements of the ring's type
template <typename Part>
int state_layers(const nvwn_engine* e, Part part)
{
    size_t off = sizeof(nvwn_slot_state_header);
    for (int l = 0; l < e->L; l++) {
        const int d = wn_score_dilation(l, e->maxDil);
        CK(part(l, off, d));
        off += (size_t)d * e->R * e->td;
    }
    return 0;
}

// Slot states at `states`, host or device memory (*host); device states need a 16-byte alignment
int check_states(const std::string& who, const void* states, bool* host)
{
    *host = !is_device_ptr(states);
    if (!*host && reinterpret_cast<uintptr_t>(states) % 16) return fail(NVWN_EINVAL, who + ": device states must be 16-byte aligned");
    return 0;
}

// Writes n slot states to `states` (host or device memory) through write(dst): device states in place, host states into the
// engine's staging buffer and from there to `states` before return.
template <typename Write>
int write_states(nvwn_engine* e, const std::string& who, void* states, int n, cudaStream_t st, Write write)
{
    bool host;
    int rc = check_states(who, states, &host);
    if (rc != 0) return rc;
    const size_t bytes = (size_t)n * wn_slot_state_bytes(*e);
    if (host) CK(e->state_stage.reserve(bytes));
    char* dst = host ? e->state_stage.get() : static_cast<char*>(states);
    if ((rc = write(dst))) return rc;
    if (host) {
        CK(cudaMemcpyAsync(states, dst, bytes, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
    }
    return 0;
}

// Before a call writes real history into rows at next_t < maxDil: from then on every launch reads the ring at every step, so the
// entries of the negative times, which no row has written since the reset, must read as the zeros of "before the start".
int clear_early_times(nvwn_engine* e, cudaStream_t st)
{
    const long long t0 = e->next_t;
    const int M = e->maxDil + 1;
    if (t0 < e->maxDil && !e->early_prime) {
        CK(e->family->clear_times(*e, e->ring, t0 - M, (int)(M - t0), st));
        e->early_prime = true;
    }
    return 0;
}

// Model v's scorer image for a scoring call of parameters p: allocated on first use, packed from the model's blob after a change
int put_score_image(nvwn_engine* e, int v, const WnParams& p, cudaStream_t st)
{
    nvwn_engine::Model& m = e->models[v];
    if (!m.score_image) CK(m.score_image.alloc(wn_score_image_bytes(e->R, e->S, e->A, e->L)));
    if (m.score_repack) {
        WnParams q = p;
        point_weights(e, q, m.blob);
        CK(wn_score_pack(m.score_image, q, st));
        m.score_repack = false;
    }
    return 0;
}

// Scoring by model: the segments of a call of Bs rows, each model it runs with its image packed, also copied to score_segs (device)
int score_segments(nvwn_engine* e, const WnParams& p, int Bs, WnScoreSegs& segs, cudaStream_t st)
{
    std::vector<int> n_of(NVWN_MAX_MODELS, 0), all_of(NVWN_MAX_MODELS, 0);
    for (int b = 0; b < e->B; b++) {
        all_of[score_model(e, b)]++;
        if (b < Bs) n_of[score_model(e, b)]++;
    }
    for (int v = 0, first = 0; v < NVWN_MAX_MODELS; first += all_of[v++]) {
        if (!n_of[v]) continue;
        const int rc = put_score_image(e, v, p, st);
        if (rc != 0) return rc;
        const nvwn_engine::Model& m = e->models[v];
        const int k = segs.count++;
        segs.model[k] = v; segs.n[k] = n_of[v]; segs.first[k] = first;
        segs.image[v] = m.score_image; segs.embPrev[v] = m.blob + e->o_embPrev; segs.embCur[v] = m.blob + e->o_embCur;
    }
    segs.order = e->score_tab;
    segs.row_model = e->score_tab + e->B;
    if (!e->score_segs) CK(e->score_segs.alloc(sizeof(WnScoreSegs)));
    return copy_snapshot(e->score_segs, &segs, 1, st);
}

}  // namespace

extern "C" {

const char* nvwn_last_error(void) { return g_err.c_str(); }

int nvwn_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

int nvwn_set_device(int device)
{
    CK(cudaSetDevice(device));
    return 0;
}

int nvwn_create(nvwn_engine** out, int dtype, int R, int S, int A, int num_layers, int max_dilation,
                int batch_size, int num_samples, int impl, int tanh_embed)
{
    if (!out) return fail(NVWN_EINVAL, "nvwn_create: out is NULL");
    *out = nullptr;
    if (dtype != NVWN_FP32 && dtype != NVWN_FP16 && dtype != NVWN_FP32_FAST) return fail(NVWN_EINVAL, "nvwn_create: dtype must be NVWN_FP32, NVWN_FP16 or NVWN_FP32_FAST");
    if (num_layers < 1 || max_dilation < 1 || batch_size < 1 || num_samples < 1) return fail(NVWN_EINVAL, "nvwn_create: sizes must be positive");
    if (!wn_stream_supported(R, S, A, dtype == NVWN_FP16))
        return fail(NVWN_EUNSUPPORTED, "nvwn_create: unsupported channel counts (R,S) must be one of (32,128) (64,128) (64,256) (128,256); A a multiple of 32");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return fail(NVWN_EUNSUPPORTED, "nvwn_create: no CUDA device (this engine has no CPU fallback)");
    }
    std::unique_ptr<nvwn_engine> e(new nvwn_engine());                 // freed with its buffers on every refusal below
    e->dtype = dtype; e->R = R; e->S = S; e->A = A; e->L = num_layers; e->maxDil = max_dilation;
    e->B = batch_size; e->N = num_samples; e->impl = impl; e->tanhEmbed = tanh_embed ? 1 : 0;
    e->td = dtype == NVWN_FP16 ? 2 : 4;
    cudaGetDevice(&e->device);
    resolve_config(*e, impl);
    e->family = e->kernel == NVWN_KERNEL_TENSORCORE ? &wn_tc_family : e->kernel == NVWN_KERNEL_LATENCY ? &wn_lat_family : &wn_stream_family;

    const size_t L = num_layers, td = e->td;
    size_t off = 0;
    auto take = [&](size_t elems) { size_t o = off; off = align_up(off + elems * td, 256); return o; };
    e->o_embPrev = take((size_t)A * R); e->o_embCur = take((size_t)A * R);
    e->o_Wprev = take(L * 2 * R * R); e->o_Wcur = take(L * 2 * R * R);
    e->o_Wres = take(L * R * R); e->o_Wskip = take(L * S * R);
    e->o_Wzs = take((size_t)A * S); e->o_Wza = take((size_t)A * A);
    e->o_Bh = take(L * 2 * R); e->o_Bres = take(L * R); e->o_Bskip = take(L * S);
    e->o_Bzs = take(A); e->o_Bza = take(A);
    e->blob_bytes = off;

    const size_t Bz = batch_size, Nz = num_samples;
    const size_t per = L * Bz * 2 * R;                                 // 64 MB of fp32 staging, or one sample of conditioning if larger
    e->stage_elems = per > ((size_t)16 << 20) ? per : ((size_t)16 << 20);
    CK(e->Lh.alloc(e->family->store_bytes(*e)));
    CK(e->sel.alloc(Nz * Bz * sizeof(float)));
    CK(e->forced.alloc(Nz * Bz * sizeof(int)));
    CK(e->yPrev.alloc(Bz * sizeof(int)));
    CK(e->yCur.alloc(Bz * sizeof(int)));
    CK(e->yOut.alloc(Nz * Bz * sizeof(int)));
    const size_t ring_bytes = e->family->ring_bytes(*e);
    CK(e->ring.alloc(ring_bytes));
    CK(e->xtOut.alloc(L * Bz * R * sizeof(float)));
    CK(e->skipOut.alloc(L * Bz * S * sizeof(float)));
    CK(e->Zs.alloc(Bz * A * sizeof(float)));
    CK(e->Za.alloc(Bz * A * sizeof(float)));
    CK(e->P.alloc(Bz * A * sizeof(float)));
    CK(e->origin.alloc(Bz * sizeof(long long)));
    CK(e->seed.alloc(Bz * sizeof(unsigned long long)));
    CK(e->slot_rows.alloc(Bz * sizeof(int)));
    CK(e->slot_seeds.alloc(Bz * sizeof(unsigned long long)));
    CK(e->prime_rows.alloc(Bz * sizeof(int)));
    if (dtype == NVWN_FP16) CK(e->stage.alloc(e->stage_elems * sizeof(float)));
    e->models.resize(NVWN_MAX_MODELS);
    e->group_rows = e->family->group_rows(*e);
    CK(e->model_tab.alloc(NVWN_MAX_MODELS * sizeof(WnModel)));
    CK(e->group_tab.alloc((Bz + e->group_rows - 1) / e->group_rows * sizeof(int)));
    const int rc = add_model(e.get(), 0);
    if (rc != 0) return rc;
    cudaMemsetAsync(e->models[0].blob, 0, e->blob_bytes, 0);
    cudaMemsetAsync(e->yOut, 0, Nz * Bz * sizeof(int), 0);
    cudaMemsetAsync(e->ring, 0, ring_bytes, 0);
    cudaMemsetAsync(e->origin, 0, Bz * sizeof(long long), 0);
    cudaMemsetAsync(e->seed, 0, Bz * sizeof(unsigned long long), 0);
    for (CondProducer* P : {&e->cond_whole, &e->cond_slots}) {
        P->T.assign(Bz, 0);
        P->start.assign(Bz, 0);
        P->live.assign(Bz, 0);
        P->first.assign(Bz, 0);
        P->done.assign(Bz, 0);
    }
    wn_fill_int(e->yPrev, 128, Bz, 0);
    wn_fill_int(e->yCur, 128, Bz, 0);
    cudaError_t se = cudaDeviceSynchronize();
    if (se != cudaSuccess) return fail((int)se, cudaGetErrorString(se));
    *out = e.release();
    return 0;
}

int nvwn_destroy(nvwn_engine* e)
{
    delete e;
    return 0;
}

int nvwn_set_embeddings(nvwn_engine* e, const float* embedPrev, const float* embedCur)
{
    if (!e || !embedPrev || !embedCur) return fail(NVWN_EINVAL, "nvwn_set_embeddings: NULL argument");
    int rc;
    if ((rc = upload(e, e->o_embPrev, embedPrev, (size_t)e->A * e->R))) return rc;
    if ((rc = upload(e, e->o_embCur, embedCur, (size_t)e->A * e->R))) return rc;
    weights_changed(e);
    CK(cudaStreamSynchronize(0));
    return 0;
}

int nvwn_set_layer_weights(nvwn_engine* e, int layer, const float* Wprev, const float* Wcur, const float* Bh,
                           const float* Wres, const float* Bres, const float* Wskip, const float* Bskip)
{
    if (!e || !Wprev || !Wcur || !Bh || !Wres || !Bres || !Wskip || !Bskip) return fail(NVWN_EINVAL, "nvwn_set_layer_weights: NULL argument");
    if (layer < 0 || layer >= e->L) return fail(NVWN_EINVAL, "nvwn_set_layer_weights: layer out of range");
    const size_t R = e->R, S = e->S, l = layer, td = e->td;
    int rc;
    if ((rc = upload(e, e->o_Wprev + l * 2 * R * R * td, Wprev, 2 * R * R))) return rc;
    if ((rc = upload(e, e->o_Wcur + l * 2 * R * R * td, Wcur, 2 * R * R))) return rc;
    if ((rc = upload(e, e->o_Bh + l * 2 * R * td, Bh, 2 * R))) return rc;
    if ((rc = upload(e, e->o_Wres + l * R * R * td, Wres, R * R))) return rc;
    if ((rc = upload(e, e->o_Bres + l * R * td, Bres, R))) return rc;
    if ((rc = upload(e, e->o_Wskip + l * S * R * td, Wskip, S * R))) return rc;
    if ((rc = upload(e, e->o_Bskip + l * S * td, Bskip, S))) return rc;
    weights_changed(e);
    CK(cudaStreamSynchronize(0));       // sources may be freed by the caller right after return
    return 0;
}

int nvwn_set_out_weights(nvwn_engine* e, const float* Wzs, const float* Bzs, const float* Wza, const float* Bza)
{
    if (!e || !Wzs || !Bzs || !Wza || !Bza) return fail(NVWN_EINVAL, "nvwn_set_out_weights: NULL argument");
    const size_t A = e->A, S = e->S;
    int rc;
    if ((rc = upload(e, e->o_Wzs, Wzs, A * S))) return rc;
    if ((rc = upload(e, e->o_Bzs, Bzs, A))) return rc;
    if ((rc = upload(e, e->o_Wza, Wza, A * A))) return rc;
    if ((rc = upload(e, e->o_Bza, Bza, A))) return rc;
    weights_changed(e);
    CK(cudaStreamSynchronize(0));
    return 0;
}

int nvwn_cond_from_features_host(float* Lh, const float* features, int batch_size, int n_cond_channels, int num_frames,
                                 const float* upsample_weight, const float* upsample_bias, int window, int stride,
                                 const float* cond_weight, const float* cond_bias, int num_layers, int R)
{
    if (!Lh || !features || !upsample_weight || !upsample_bias || !cond_weight || !cond_bias) return fail(NVWN_EINVAL, "nvwn_cond_from_features_host: NULL argument");
    if (batch_size < 1 || n_cond_channels < 1 || num_frames < 1 || window < stride || stride < 1 || num_layers < 1 || R < 1)
        return fail(NVWN_EINVAL, "nvwn_cond_from_features_host: bad sizes (need window >= stride >= 1)");
    wn_cond_host(Lh, features, upsample_weight, upsample_bias, cond_weight, cond_bias, batch_size, n_cond_channels, num_frames, window, stride, num_layers, R);
    return 0;
}

int nvwn_cond_producer_load(nvwn_engine* e, const float* features, int n_cond_channels, int num_frames,
                            const float* upsample_weight, const float* upsample_bias, int window, int stride,
                            const float* cond_weight, const float* cond_bias, void* stream)
{
    const std::string who = "nvwn_cond_producer_load";
    if (!e || !features || !upsample_weight || !upsample_bias || !cond_weight || !cond_bias) return fail(NVWN_EINVAL, who + ": NULL argument");
    const int C = n_cond_channels, T = num_frames, K = window;
    int rc = check_cond_sizes(who, C, K, stride);
    if (rc != 0) return rc;
    if (T < 1) return fail(NVWN_EINVAL, who + ": num_frames = " + std::to_string(T) + "; need >= 1");
    cudaStream_t st = (cudaStream_t)stream;
    CondProducer& P = e->cond_whole;
    P.T.assign(e->B, 0);                                                      // loaded once every copy has been made
    P.ring = 0;                                                               // ends a live sequence
    if ((rc = put_cond_network(e, P, who, C, K, stride, upsample_weight, upsample_bias, cond_weight, cond_bias, st))) return rc;
    // features [B][C][T] are the frame arena with cap = T, in one copy; row b's utterance starts at sample 0
    const size_t n_feat = (size_t)e->B * C * T;
    CK(P.frames.reserve(n_feat * sizeof(float)));
    P.cap = T;
    std::vector<WnCondSlot> tab(e->B);
    for (int b = 0; b < e->B; b++) tab[b] = cond_row(P, b, T);
    cudaError_t ce = cudaMemcpyAsync(P.frames, features, n_feat * sizeof(float), cudaMemcpyDefault, st);
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(P.tables + cond_table_offset(e), tab.data(), tab.size() * sizeof(WnCondSlot), cudaMemcpyHostToDevice, st);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);                   // host sources may be released by the caller now
    if (ce != cudaSuccess) return fail((int)ce, who + ": " + cudaGetErrorString(ce));
    P.T.assign(e->B, T);
    return 0;
}

int nvwn_cond_producer_run(nvwn_engine* e, int first_sample, int sample_begin, int sample_count, void* stream)
{
    if (!e) return fail(NVWN_EINVAL, "nvwn_cond_producer_run: NULL engine");
    const CondProducer& P = e->cond_whole;
    if (P.ring) return fail(NVWN_EINVAL, "nvwn_cond_producer_run: a live sequence is produced with nvwn_cond_producer_run_stream");
    if (P.T[0] < 1) return fail(NVWN_EINVAL, "nvwn_cond_producer_run: nvwn_cond_producer_load has not been called");
    const long long Nn = (long long)P.T[0] * P.stride;
    if (sample_begin < 0 || sample_count < 0 || sample_begin + (long long)sample_count > Nn) return fail(NVWN_EINVAL, "nvwn_cond_producer_run: sample range outside num_frames * stride");
    if (first_sample < 0 || first_sample + (long long)sample_begin + sample_count > e->N) return fail(NVWN_EINVAL, "nvwn_cond_producer_run: samples do not fit the engine");
    return produce(e, P, "nvwn_cond_producer", nullptr, e->B, sample_begin, first_sample + sample_begin, sample_count, (cudaStream_t)stream);
}

int nvwn_cond_producer_run_stream(nvwn_engine* e, long long sample_begin, int sample_count, void* stream)
{
    const std::string who = "nvwn_cond_producer_run_stream";
    if (!e) return fail(NVWN_EINVAL, who + ": NULL engine");
    CondProducer& P = e->cond_whole;
    if (P.T[0] < 1 && !P.ring) return fail(NVWN_EINVAL, who + ": nvwn_cond_producer_load has not been called");
    const long long Nn = (long long)P.T[0] * P.stride;
    if (sample_begin < 0 || sample_count < 0 || sample_begin + sample_count > Nn)
        return fail(NVWN_EINVAL, P.ring ? who + ": samples [" + std::to_string(sample_begin) + ", " + std::to_string(sample_begin + sample_count) +
                                             ") of the live sequence are not all below the " + std::to_string(Nn) + " its " + std::to_string(P.T[0]) +
                                             " pushed frames give"
                                        : who + ": sample range outside num_frames * stride");
    int rc = check_window(e, who, sample_begin, sample_count, "sample_count", 0);
    if (rc != 0) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (P.ring && sample_count > 0) {
        // the first frame the range reads must still be in the ring; every row holds the same frames
        rc = check_held(P, who, 0, sample_begin, "");
        if (rc != 0) return rc;
        if ((rc = put_cond_table(e, P, nullptr, e->B, st))) return rc;
        mark_produced(P, nullptr, e->B, sample_begin + sample_count);
    }
    for (const WrapPiece& w : split_at_wrap(sample_begin, sample_count, e->N)) {
        rc = produce(e, P, "nvwn_cond_producer", nullptr, e->B, sample_begin + w.off, w.pos, w.len, st);
        if (rc != 0) return rc;
    }
    return 0;
}

int nvwn_cond_producer_open_live(nvwn_engine* e, int n_cond_channels, const float* upsample_weight, const float* upsample_bias, int window, int stride,
                                 const float* cond_weight, const float* cond_bias, int ring_frames, void* stream)
{
    const std::string who = "nvwn_cond_producer_open_live";
    if (!e || !upsample_weight || !upsample_bias || !cond_weight || !cond_bias) return fail(NVWN_EINVAL, who + ": NULL argument");
    int rc = check_cond_sizes(who, n_cond_channels, window, stride);
    if (rc == 0) rc = check_ring_frames(who, ring_frames, window, stride);
    if (rc != 0) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    CondProducer& P = e->cond_whole;
    P.T.assign(e->B, 0);                                                      // replaces a loaded sequence
    P.ring = 0;
    if ((rc = put_cond_network(e, P, who, n_cond_channels, window, stride, upsample_weight, upsample_bias, cond_weight, cond_bias, st))) return rc;
    CK(P.frames.reserve((size_t)e->B * n_cond_channels * ring_frames * sizeof(float)));
    const cudaError_t ce = cudaStreamSynchronize(st);                        // host sources may be released by the caller now
    if (ce != cudaSuccess) return fail((int)ce, who + ": " + cudaGetErrorString(ce));
    P.cap = P.ring = ring_frames;
    P.done.assign(e->B, 0);
    return 0;
}

int nvwn_cond_producer_push(nvwn_engine* e, const float* features, int num_frames, void* stream)
{
    const std::string who = "nvwn_cond_producer_push";
    if (!e) return fail(NVWN_EINVAL, who + ": NULL engine");
    CondProducer& P = e->cond_whole;
    if (!P.ring) return fail(NVWN_EINVAL, who + ": no live sequence is open (nvwn_cond_producer_open_live; nvwn_cond_producer_load ends one)");
    if (num_frames < 0) return fail(NVWN_EINVAL, who + ": num_frames = " + std::to_string(num_frames) + " < 0");
    if (num_frames == 0) return 0;
    if (!features) return fail(NVWN_EINVAL, who + ": features is NULL");
    const long long T = P.T[0], T1 = T + num_frames;
    if (T1 * P.stride > INT_MAX)
        return fail(NVWN_EINVAL, who + ": a live sequence holds at most INT_MAX samples; " + std::to_string(T1) + " frames would give " +
                                     std::to_string(T1 * P.stride));
    int rc = check_push(P, who, 0, num_frames, "");                          // every row holds the same frames
    if (rc == 0) rc = put_live_frames(P, 0, e->B, T, features, num_frames, (cudaStream_t)stream);
    if (rc != 0) return rc;
    P.T.assign(e->B, (int)T1);
    return 0;
}

int nvwn_set_conditioning_from_features(nvwn_engine* e, const float* features, int n_cond_channels, int num_frames,
                                        const float* upsample_weight, const float* upsample_bias, int window, int stride,
                                        const float* cond_weight, const float* cond_bias, int first_sample, void* stream)
{
    if (!e) return fail(NVWN_EINVAL, "nvwn_set_conditioning_from_features: NULL argument");
    const long long Nn = (long long)num_frames * stride;
    if (first_sample < 0 || (num_frames >= 1 && stride >= 1 && first_sample + Nn > e->N)) return fail(NVWN_EINVAL, "nvwn_set_conditioning_from_features: num_frames * stride samples do not fit the engine");
    int rc = nvwn_cond_producer_load(e, features, n_cond_channels, num_frames, upsample_weight, upsample_bias, window, stride, cond_weight, cond_bias, stream);
    if (rc != 0) return rc;
    rc = nvwn_cond_producer_run(e, first_sample, 0, (int)Nn, stream);
    if (rc != 0) return rc;
    CK(cudaStreamSynchronize((cudaStream_t)stream));                        // "returns after the work has completed"
    return 0;
}

int nvwn_cond_producer_set_weights(nvwn_engine* e, int n_cond_channels, const float* upsample_weight, const float* upsample_bias, int window,
                                   int stride, const float* cond_weight, const float* cond_bias, void* stream)
{
    const std::string who = "nvwn_cond_producer_set_weights";
    if (!e || !upsample_weight || !upsample_bias || !cond_weight || !cond_bias) return fail(NVWN_EINVAL, who + ": NULL argument");
    const int C = n_cond_channels;
    int rc = check_cond_sizes(who, C, window, stride);
    if (rc != 0) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    CondProducer& P = e->cond_slots;
    if (P.frames && C != P.C) {                                               // the arena is laid out for the old channel count
        CK(cudaDeviceSynchronize());
        P.frames = DevBuf<float>();
        P.cap = 0;
    }
    P.T.assign(e->B, 0);                                                      // frames attached under the old network are forgotten
    P.live.assign(e->B, 0);                                                   // and live mode ends
    P.ring = 0;
    if ((rc = put_cond_network(e, P, who, C, window, stride, upsample_weight, upsample_bias, cond_weight, cond_bias, st))) return rc;
    const cudaError_t ce = cudaStreamSynchronize(st);                        // host sources may be released by the caller now
    if (ce != cudaSuccess) return fail((int)ce, who + ": " + cudaGetErrorString(ce));
    return 0;
}

int nvwn_cond_producer_set_slots(nvwn_engine* e, const int* slots, int n, const float* const* features, const int* num_frames,
                                 const long long* starts, void* stream)
{
    const std::string who = "nvwn_cond_producer_set_slots";
    if (!e) return fail(NVWN_EINVAL, who + ": NULL engine");
    CondProducer& P = e->cond_slots;
    if (!P.scratch) return fail(NVWN_EINVAL, who + ": nvwn_cond_producer_set_weights has not been called");
    if (P.ring)
        return fail(NVWN_EINVAL, who + ": the per-slot producer is in live mode (nvwn_cond_producer_open_live_slots; nvwn_cond_producer_set_weights and "
                                       "nvwn_reset_history end it)");
    int rc = check_slots(e, who, slots, n);
    if (rc != 0) return rc;
    if (!features || !num_frames || !starts) return fail(NVWN_EINVAL, who + ": features, num_frames or starts is NULL");
    const int C = P.C;
    int most = 0;
    for (int i = 0; i < n; i++) {
        const std::string u = "utterance " + std::to_string(i) + " (slot " + std::to_string(slots[i]) + ")";
        if (!features[i]) return fail(NVWN_EINVAL, who + ": the frames of " + u + " are NULL");
        if (num_frames[i] < 1) return fail(NVWN_EINVAL, who + ": " + u + " has num_frames = " + std::to_string(num_frames[i]) + "; need >= 1");
        if ((long long)num_frames[i] * P.stride > INT_MAX) return fail(NVWN_EINVAL, who + ": " + u + " has more than INT_MAX samples");
        if (starts[i] < 0) return fail(NVWN_EINVAL, who + ": " + u + " starts at " + std::to_string(starts[i]) + " < 0");
        if (num_frames[i] > most) most = num_frames[i];
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (most > P.cap) {
        // a larger arena; the frames of the other slots move with it
        const int cap = most > 2 * P.cap ? most : 2 * P.cap;
        DevBuf<float> grown;
        CK(grown.alloc((size_t)e->B * cap * C * sizeof(float)));
        if (P.frames) {
            const size_t old_pitch = (size_t)P.cap * C * sizeof(float);
            cudaError_t ce = cudaMemcpy2DAsync(grown, (size_t)cap * C * sizeof(float), P.frames, old_pitch, old_pitch, e->B, cudaMemcpyDeviceToDevice, st);
            if (ce == cudaSuccess) ce = cudaDeviceSynchronize();             // no launch reads the old arena any more
            if (ce != cudaSuccess) return fail((int)ce, who + ": " + cudaGetErrorString(ce));
        }
        P.frames = std::move(grown);
        P.cap = cap;
    }
    for (int i = 0; i < n; i++) {
        float* dst = P.frames + (size_t)slots[i] * P.cap * C;
        const size_t count = (size_t)C * num_frames[i];
        if (is_device_ptr(features[i])) CK(cudaMemcpyAsync(dst, features[i], count * sizeof(float), cudaMemcpyDeviceToDevice, st));
        else if ((rc = copy_snapshot(dst, features[i], count, st))) return rc;     // staged: the caller may reuse its memory on return
    }
    for (int i = 0; i < n; i++) {
        P.T[slots[i]] = num_frames[i];
        P.start[slots[i]] = starts[i];
    }
    e->slot_rows_used = true;
    return 0;
}

int nvwn_cond_producer_run_slots(nvwn_engine* e, const int* slots, int n, long long first_sample, int num_samples, void* stream)
{
    const std::string who = "nvwn_cond_producer_run_slots";
    if (!e) return fail(NVWN_EINVAL, who + ": NULL engine");
    CondProducer& P = e->cond_slots;
    if (!P.scratch) return fail(NVWN_EINVAL, who + ": nvwn_cond_producer_set_weights has not been called");
    int rc = check_slots(e, who, slots, n);
    if (rc == 0) rc = check_window(e, who, first_sample, num_samples, "num_samples", 0);
    if (rc != 0) return rc;
    for (int i = 0; i < n; i++) {
        const int s = slots[i];
        if (P.ring ? !P.live[s] : P.T[s] < 1)
            return fail(NVWN_EINVAL, who + ": slot " + std::to_string(s) +
                                         (P.ring ? " has no live utterance attached (nvwn_cond_producer_attach_live)"
                                                 : " has no frames attached (nvwn_cond_producer_set_slots; nvwn_reset_history and nvwn_cond_producer_set_weights "
                                                   "forget them)"));
        if (first_sample < P.start[s])
            return fail(NVWN_EINVAL, who + ": first_sample " + std::to_string(first_sample) + " is before the start " + std::to_string(P.start[s]) +
                                         " of slot " + std::to_string(s) + "'s utterance");
        // the range's first sample reads the earliest frames of the range
        const long long n0 = first_sample - P.start[s];
        if (P.ring && num_samples > 0 && n0 < (long long)P.T[s] * P.stride &&
            (rc = check_held(P, who, s, n0, " of slot " + std::to_string(s) + "'s utterance")))
            return rc;
    }
    e->slot_rows_used = true;
    if (P.ring && num_samples > 0) mark_produced(P, slots, n, first_sample + num_samples);
    if (num_samples == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    if ((rc = put_cond_table(e, P, slots, n, st))) return rc;
    for (const WrapPiece& w : split_at_wrap(first_sample, num_samples, e->N))
        if ((rc = produce(e, P, who, slots, n, first_sample + w.off, w.pos, w.len, st))) return rc;
    return 0;
}

int nvwn_cond_producer_open_live_slots(nvwn_engine* e, int ring_frames, void* stream)
{
    const std::string who = "nvwn_cond_producer_open_live_slots";
    (void)stream;                                                             // nothing is enqueued: the rings fill with the pushes
    if (!e) return fail(NVWN_EINVAL, who + ": NULL engine");
    CondProducer& P = e->cond_slots;
    if (!P.scratch) return fail(NVWN_EINVAL, who + ": nvwn_cond_producer_set_weights has not been called");
    const int rc = check_ring_frames(who, ring_frames, P.K, P.stride);
    if (rc != 0) return rc;
    CK(P.frames.reserve((size_t)e->B * P.C * ring_frames * sizeof(float)));
    P.cap = P.ring = ring_frames;
    P.T.assign(e->B, 0);
    P.live.assign(e->B, 0);
    return 0;
}

int nvwn_cond_producer_attach_live(nvwn_engine* e, const int* slots, int n, const long long* starts, const int* first_frames,
                                   const float* const* features, const int* num_frames, void* stream)
{
    const std::string who = "nvwn_cond_producer_attach_live";
    if (!e) return fail(NVWN_EINVAL, who + ": NULL engine");
    CondProducer& P = e->cond_slots;
    if (!P.ring) return fail(NVWN_EINVAL, who + ": the per-slot producer is not in live mode (nvwn_cond_producer_open_live_slots)");
    int rc = check_slots(e, who, slots, n);
    if (rc != 0) return rc;
    if (!starts || !first_frames || !num_frames) return fail(NVWN_EINVAL, who + ": starts, first_frames or num_frames is NULL");
    for (int i = 0; i < n; i++) {
        const std::string u = "utterance " + std::to_string(i) + " (slot " + std::to_string(slots[i]) + ")";
        if (first_frames[i] < 0 || num_frames[i] < 0 || num_frames[i] > P.ring)
            return fail(NVWN_EINVAL, who + ": " + u + " has first_frames = " + std::to_string(first_frames[i]) + " and num_frames = " +
                                         std::to_string(num_frames[i]) + "; need first_frames >= 0 and 0 <= num_frames <= ring_frames (" +
                                         std::to_string(P.ring) + ")");
        if (num_frames[i] > 0 && (!features || !features[i])) return fail(NVWN_EINVAL, who + ": the frames of " + u + " are NULL");
        if (((long long)first_frames[i] + num_frames[i]) * P.stride > INT_MAX) return fail(NVWN_EINVAL, who + ": " + u + " has more than INT_MAX samples");
    }
    cudaStream_t st = (cudaStream_t)stream;
    for (int i = 0; i < n; i++)
        if (num_frames[i] > 0 && (rc = put_live_frames(P, slots[i], 1, first_frames[i], features[i], num_frames[i], st))) return rc;
    for (int i = 0; i < n; i++) {
        const int s = slots[i];
        P.live[s] = 1;
        P.first[s] = first_frames[i];
        P.T[s] = first_frames[i] + num_frames[i];
        P.start[s] = starts[i];
        P.done[s] = 0;
    }
    e->slot_rows_used = true;
    return 0;
}

int nvwn_cond_producer_push_slots(nvwn_engine* e, const int* slots, int n, const float* const* features, const int* num_frames, void* stream)
{
    const std::string who = "nvwn_cond_producer_push_slots";
    if (!e) return fail(NVWN_EINVAL, who + ": NULL engine");
    CondProducer& P = e->cond_slots;
    if (!P.ring) return fail(NVWN_EINVAL, who + ": the per-slot producer is not in live mode (nvwn_cond_producer_open_live_slots)");
    int rc = check_slots(e, who, slots, n);
    if (rc != 0) return rc;
    if (!features || !num_frames) return fail(NVWN_EINVAL, who + ": features or num_frames is NULL");
    for (int i = 0; i < n; i++) {
        const int s = slots[i];
        const std::string u = "slot " + std::to_string(s);
        if (!P.live[s]) return fail(NVWN_EINVAL, who + ": " + u + " has no live utterance attached (nvwn_cond_producer_attach_live)");
        if (num_frames[i] < 0) return fail(NVWN_EINVAL, who + ": num_frames = " + std::to_string(num_frames[i]) + " < 0 for " + u);
        if (num_frames[i] > 0 && !features[i]) return fail(NVWN_EINVAL, who + ": the frames of " + u + " are NULL");
        const long long T1 = (long long)P.T[s] + num_frames[i];
        if (T1 * P.stride > INT_MAX) return fail(NVWN_EINVAL, who + ": " + u + "'s utterance would hold more than INT_MAX samples");
        rc = check_push(P, who, s, num_frames[i], " of " + u);
        if (rc != 0) return rc;
    }
    cudaStream_t st = (cudaStream_t)stream;
    for (int i = 0; i < n; i++) {
        if (num_frames[i] == 0) continue;
        if ((rc = put_live_frames(P, slots[i], 1, P.T[slots[i]], features[i], num_frames[i], st))) return rc;
        P.T[slots[i]] += num_frames[i];
    }
    return 0;
}

int nvwn_reset_history(nvwn_engine* e)
{
    if (!e) return fail(NVWN_EINVAL, "nvwn_reset_history: NULL engine");
    CK(wn_fill_int(e->yPrev, 128, e->B, 0));      // silenceInputs, nv_wavenet.cuh:213-218
    CK(wn_fill_int(e->yCur, 128, e->B, 0));
    CK(cudaMemsetAsync(e->origin, 0, (size_t)e->B * sizeof(long long), 0));
    CK(cudaMemsetAsync(e->seed, 0, (size_t)e->B * sizeof(unsigned long long), 0));
    e->next_t = 0;
    e->slot_rows_used = false;
    e->prime_bs = 0;
    e->early_prime = false;
    e->cond_slots.T.assign(e->B, 0);              // attached frames: their starts are absolute samples of the old timeline
    e->cond_slots.live.assign(e->B, 0);           // and the per-slot producer's live mode ends
    e->cond_slots.ring = 0;
    return 0;
}

int nvwn_restart_slots(nvwn_engine* e, const int* slots, int n, const unsigned long long* seeds, void* stream)
{
    if (!e) return fail(NVWN_EINVAL, "nvwn_restart_slots: NULL engine");
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned long long* seeds_dev;
    const int rc = take_slots(e, "nvwn_restart_slots", slots, n, seeds, &seeds_dev, st);
    if (rc != 0) return rc;
    // a zero history row and silence fed back are exactly the state of a fresh start (DESIGN.md §6)
    CK(e->family->clear_rows(*e, e->ring, e->slot_rows, n, st));
    CK(wn_restart_rows(e->slot_rows, n, seeds_dev, e->next_t, e->yPrev, e->yCur, e->origin, e->seed, st));
    return 0;
}

int nvwn_set_conditioning_slots(nvwn_engine* e, const float* Lh, const int* slots, int n, long long first_sample, int num_samples, void* stream)
{
    const std::string who = "nvwn_set_conditioning_slots";
    if (!e) return fail(NVWN_EINVAL, who + ": NULL engine");
    if (!Lh) return fail(NVWN_EINVAL, who + ": Lh is NULL");
    cudaStream_t st = (cudaStream_t)stream;
    int rc = check_window(e, who, first_sample, num_samples, "num_samples", 0);
    if (rc == 0) rc = take_slots(e, who, slots, n, nullptr, nullptr, st);
    if (rc != 0) return rc;
    const size_t unit = (size_t)e->L * n * 2 * e->R;                        // floats per sample
    for (const WrapPiece& w : split_at_wrap(first_sample, num_samples, e->N)) {
        rc = feed(e, Lh + (size_t)w.off * unit, (size_t)w.len, unit, true, st, [&](const float* s, size_t first, size_t m) {
            return e->family->convert_rows(*e, e->Lh, s, e->slot_rows, n, w.pos + (int)first, (int)m, st);
        });
        if (rc != 0) return rc;
    }
    return 0;
}

int nvwn_set_selectors_random_slots(nvwn_engine* e, long long first_sample, int num_samples, void* stream)
{
    if (!e) return fail(NVWN_EINVAL, "nvwn_set_selectors_random_slots: NULL engine");
    const int rc = check_window(e, "nvwn_set_selectors_random_slots", first_sample, num_samples, "num_samples", 0);
    if (rc != 0) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t B = e->B;
    e->slot_rows_used = true;
    for (const WrapPiece& w : split_at_wrap(first_sample, num_samples, e->N))
        CK(wn_fill_selectors_slots(e->sel + (size_t)w.pos * B, w.len, e->B, first_sample + w.off, e->origin, e->seed, st));
    return 0;
}

int nvwn_set_selectors(nvwn_engine* e, const float* selectors)
{
    if (!e || !selectors) return fail(NVWN_EINVAL, "nvwn_set_selectors: NULL argument");
    CK(cudaMemcpy(e->sel, selectors, (size_t)e->N * e->B * sizeof(float), cudaMemcpyDefault));
    return 0;
}

int nvwn_libc_selectors(float* selectors, int batch_size, int sample_count)
{
    if (!selectors || batch_size < 1 || sample_count < 1) return fail(NVWN_EINVAL, "nvwn_libc_selectors: bad argument");
    // Matrix outputSelectors(batch_size, sample_count); outputSelectors.randomize(0.5, 1.0)  (pytorch/wavenet_infer.cu:92-93,
    // matrix.cpp:38-56): rows = batch visited outermost, two rand() per element, column-major storage
    for (int b = 0; b < batch_size; b++) {
        for (int s = 0; s < sample_count; s++) {
            (void)(rand() % 100);                                   // sparsity draw (sparsity = 0)
            float r = static_cast<float>(rand()) / static_cast<float>(RAND_MAX);
            r -= 0.5;
            r = r * 1.0f + 0.5f;
            selectors[(size_t)s * batch_size + b] = r;
        }
    }
    return 0;
}

int nvwn_set_selectors_random(nvwn_engine* e, unsigned long long seed, void* stream)
{
    if (!e) return fail(NVWN_EINVAL, "nvwn_set_selectors_random: NULL engine");
    CK(wn_fill_selectors(e->sel, (size_t)e->N * e->B, seed, 0, (cudaStream_t)stream));
    return 0;
}

int nvwn_set_selectors_random_stream(nvwn_engine* e, unsigned long long seed, long long first_sample, int num_samples, void* stream)
{
    if (!e) return fail(NVWN_EINVAL, "nvwn_set_selectors_random_stream: NULL engine");
    const int rc = check_window(e, "nvwn_set_selectors_random_stream", first_sample, num_samples, "num_samples", 0);
    if (rc != 0) return rc;
    const size_t B = e->B;
    for (const WrapPiece& w : split_at_wrap(first_sample, num_samples, e->N))
        CK(wn_fill_selectors(e->sel + (size_t)w.pos * B, (size_t)w.len * B, seed, (unsigned long long)(first_sample + w.off) * B, (cudaStream_t)stream));
    return 0;
}

int nvwn_set_conditioning(nvwn_engine* e, const float* Lh, int first_sample, int num_samples, void* stream)
{
    if (!e || !Lh) return fail(NVWN_EINVAL, "nvwn_set_conditioning: NULL argument");
    if (first_sample < 0 || num_samples < 0 || first_sample + num_samples > e->N) return fail(NVWN_EINVAL, "nvwn_set_conditioning: sample range out of bounds");
    cudaStream_t st = (cudaStream_t)stream;
    return feed(e, Lh, num_samples, (size_t)e->L * e->B * 2 * e->R, false, st, [&](const float* src, size_t first, size_t m) {
        return e->family->convert(*e, e->Lh, src, first_sample + (int)first, (int)m, st);
    });
}

int nvwn_set_inputs(nvwn_engine* e, const float* Lh, const float* selectors)
{
    if (!e || !Lh || !selectors) return fail(NVWN_EINVAL, "nvwn_set_inputs: NULL argument");
    int rc;
    if ((rc = nvwn_reset_history(e))) return rc;
    if ((rc = nvwn_set_conditioning(e, Lh, 0, e->N, nullptr))) return rc;
    if ((rc = nvwn_set_selectors(e, selectors))) return rc;
    CK(cudaStreamSynchronize(0));
    return 0;
}

int nvwn_set_forced(nvwn_engine* e, const int* forced)
{
    if (!e) return fail(NVWN_EINVAL, "nvwn_set_forced: NULL engine");
    if (!forced) { e->use_forced = false; return 0; }
    CK(cudaMemcpy(e->forced, forced, (size_t)e->N * e->B * sizeof(int), cudaMemcpyDefault));
    e->use_forced = true;
    return 0;
}

int nvwn_weight_blob(nvwn_engine* e, void** dev_ptr, unsigned long long* bytes)
{
    if (!e || !dev_ptr || !bytes) return fail(NVWN_EINVAL, "nvwn_weight_blob: NULL argument");
    *dev_ptr = e->models[0].blob;
    *bytes = e->blob_bytes;
    return 0;
}

int nvwn_weights_updated(nvwn_engine* e)
{
    if (!e) return fail(NVWN_EINVAL, "nvwn_weights_updated: NULL engine");
    weights_changed(e);
    return 0;
}

int nvwn_set_model(nvwn_engine* e, int model, const nvwn_engine* src)
{
    const std::string who = "nvwn_set_model";
    if (!e || !src) return fail(NVWN_EINVAL, who + ": NULL engine");
    if (model < 1 || model >= NVWN_MAX_MODELS)
        return fail(NVWN_EINVAL, who + ": model " + std::to_string(model) + " is outside [1, " + std::to_string(NVWN_MAX_MODELS) +
                                       ") (model 0 is the engine's own weights: use the setters)");
    if (src->dtype != e->dtype || src->R != e->R || src->S != e->S || src->A != e->A || src->L != e->L || src->maxDil != e->maxDil ||
        src->tanhEmbed != e->tanhEmbed || src->device != e->device)
        return fail(NVWN_EINVAL, who + ": the source engine differs in dtype, R, S, A, L, max_dilation, tanh_embed or device");
    // first set: the buffers, and the model's entry of the base table, which no launch reads before a group names the model
    int rc;
    if (!e->models[model].blob && (rc = add_model(e, model))) return rc;
    CK(cudaMemcpyAsync(e->models[model].blob, src->models[0].blob, e->blob_bytes, cudaMemcpyDeviceToDevice, 0));
    model_changed(e, model);
    if (e->score_next >= 0)                  // an open scoring stream whose rows run the model ends, as at a weight change
        for (int b = 0; b < e->score_bs; b++)
            if (score_model(e, b) == model) { e->score_next = -1; break; }
    CK(cudaStreamSynchronize(0));       // src may be changed or destroyed on return
    return 0;
}

int nvwn_model_group(nvwn_engine* e, int* rows)
{
    if (!e || !rows) return fail(NVWN_EINVAL, "nvwn_model_group: NULL argument");
    *rows = e->group_rows;
    return 0;
}

int nvwn_set_group_models(nvwn_engine* e, const int* models, int n_groups, void* stream)
{
    const std::string who = "nvwn_set_group_models";
    if (!e || !models) return fail(NVWN_EINVAL, who + ": NULL argument");
    const int groups = (e->B + e->group_rows - 1) / e->group_rows;
    if (n_groups != groups)
        return fail(NVWN_EINVAL, who + ": need n_groups = ceil(B / G) = " + std::to_string(groups) + " (G = " + std::to_string(e->group_rows) + "); got " +
                                       std::to_string(n_groups));
    int rc = check_models(e, who, "group", models, n_groups);
    if (rc == 0) rc = copy_snapshot(e->group_tab, models, n_groups, (cudaStream_t)stream);
    if (rc != 0) return rc;
    e->group_host.assign(models, models + n_groups);
    return 0;
}

int nvwn_set_score_models(nvwn_engine* e, const int* models, int n_rows, void* stream)
{
    const std::string who = "nvwn_set_score_models";
    if (!e || !models) return fail(NVWN_EINVAL, who + ": NULL argument");
    if (e->dtype != NVWN_FP16) return fail(NVWN_EUNSUPPORTED, who + ": only NVWN_FP16 engines can score");
    if (n_rows != e->B) return fail(NVWN_EINVAL, who + ": need n_rows = B = " + std::to_string(e->B) + "; got " + std::to_string(n_rows));
    int rc = check_models(e, who, "row", models, n_rows);
    if (rc != 0) return rc;
    // the rows by model, then by row, and the table: a call of Bs rows takes of each model's rows the prefix below Bs
    std::vector<int> tab(2 * (size_t)n_rows);
    size_t k = 0;
    for (int v = 0; v < NVWN_MAX_MODELS; v++)
        for (int b = 0; b < n_rows; b++)
            if (models[b] == v) tab[k++] = b;
    std::copy(models, models + n_rows, tab.begin() + n_rows);
    if (!e->score_tab) CK(e->score_tab.alloc(tab.size() * sizeof(int)));
    rc = copy_snapshot(e->score_tab, tab.data(), tab.size(), (cudaStream_t)stream);
    if (rc != 0) return rc;
    e->score_models.assign(models, models + n_rows);
    e->score_next = -1;                      // the open stream's fronts were computed with the old models
    return 0;
}

int nvwn_run_partial(nvwn_engine* e, int init_sample, int count, int num_samples, int batch_size,
                     int* yOut, int dump_activations, void* stream_)
{
    if (!e) return fail(NVWN_EINVAL, "nvwn_run_partial: NULL engine");
    if (batch_size < 1 || batch_size > e->B || num_samples < 1 || num_samples > e->N)
        return fail(NVWN_EINVAL, "nvwn_run_partial: batch_size / num_samples exceed what the engine was created for");
    if (init_sample < 0 || count < 0 || init_sample + count > num_samples) return fail(NVWN_EINVAL, "nvwn_run_partial: sample range out of bounds");
    cudaStream_t stream = (cudaStream_t)stream_;
    const int rc = launch_steps(e, "nvwn_run_partial", init_sample, init_sample, count, num_samples, batch_size, dump_activations ? 1 : 0, stream);
    if (rc != 0) return rc;
    if (yOut) CK(cudaMemcpyAsync(yOut, e->yOut, (size_t)num_samples * batch_size * sizeof(int), cudaMemcpyDefault, stream));
    return 0;
}

int nvwn_run_stream(nvwn_engine* e, long long first_sample, int count, int batch_size, int dump_activations, void* stream_)
{
    if (!e) return fail(NVWN_EINVAL, "nvwn_run_stream: NULL engine");
    if (batch_size < 1 || batch_size > e->B) return fail(NVWN_EINVAL, "nvwn_run_stream: batch_size outside [1, B] of the engine");
    int rc = check_window(e, "nvwn_run_stream", first_sample, count, "count", 0);
    if (rc != 0) return rc;
    if (first_sample != e->next_t)
        return fail(NVWN_EINVAL, "nvwn_run_stream: first_sample " + std::to_string(first_sample) + " does not continue the utterance batch: the next sample is " +
                                     std::to_string(e->next_t) + " (nvwn_reset_history starts over at 0)");
    cudaStream_t stream = (cudaStream_t)stream_;
    const int dump = dump_activations ? 1 : 0;
    for (const WrapPiece& w : split_at_wrap(first_sample, count, e->N))
        if ((rc = launch_steps(e, "nvwn_run_stream", w.pos, first_sample + w.off, w.len, e->N, batch_size, w.off + w.len == count ? dump : 0, stream)))
            return rc;
    return 0;
}

int nvwn_run(nvwn_engine* e, int num_samples, int batch_size, int* yOut, int dump_activations, void* stream)
{
    return nvwn_run_partial(e, 0, num_samples, num_samples, batch_size, yOut, dump_activations, stream);
}

int nvwn_get_yout(nvwn_engine* e, int* yOut, int offset, int size, void* stream)
{
    if (!e || !yOut) return fail(NVWN_EINVAL, "nvwn_get_yout: NULL argument");
    if (offset < 0 || size < 0 || offset + size > e->N) return fail(NVWN_EINVAL, "nvwn_get_yout: range out of bounds");
    if (size == 0) return 0;
    const size_t pitch = (size_t)e->N * sizeof(int);
    CK(cudaMemcpy2DAsync(yOut + offset, pitch, e->yOut + offset, pitch, (size_t)size * sizeof(int), e->B, cudaMemcpyDefault, (cudaStream_t)stream));
    return 0;
}

int nvwn_get_xt_out(nvwn_engine* e, int layer, float* out)
{
    if (!e || !out || layer < 0 || layer >= e->L) return fail(NVWN_EINVAL, "nvwn_get_xt_out: bad argument");
    return download(out, e->xtOut + (size_t)layer * e->B * e->R, (size_t)e->B * e->R);
}
int nvwn_get_skip_out(nvwn_engine* e, int layer, float* out)
{
    if (!e || !out || layer < 0 || layer >= e->L) return fail(NVWN_EINVAL, "nvwn_get_skip_out: bad argument");
    return download(out, e->skipOut + (size_t)layer * e->B * e->S, (size_t)e->B * e->S);
}
int nvwn_get_zs(nvwn_engine* e, float* out) { return (!e || !out) ? fail(NVWN_EINVAL, "nvwn_get_zs: NULL") : download(out, e->Zs, (size_t)e->B * e->A); }
int nvwn_get_za(nvwn_engine* e, float* out) { return (!e || !out) ? fail(NVWN_EINVAL, "nvwn_get_za: NULL") : download(out, e->Za, (size_t)e->B * e->A); }
int nvwn_get_p(nvwn_engine* e, float* out) { return (!e || !out) ? fail(NVWN_EINVAL, "nvwn_get_p: NULL") : download(out, e->P, (size_t)e->B * e->A); }

// mu-law expansion of one code, exactly as the reference's post-processing does it in double precision
// (pytorch/utils.py:62-70 mu_law_decode_numpy, called with mu_quantization = A by pytorch/nv_wavenet_inference.py:58):
//   mu = A - 1;  signal = 2 (x / mu) - 1;  audio = sign(signal) (1 / mu) ((1 + mu)^|signal| - 1)
static double mulaw_expand(int x, int A)
{
    const double mu = (double)A - 1.0;
    const double signal = 2.0 * ((double)x / mu) - 1.0;
    const double magnitude = (1.0 / mu) * (pow(1.0 + mu, fabs(signal)) - 1.0);
    return signal > 0.0 ? magnitude : (signal < 0.0 ? -magnitude : 0.0);
}

int nvwn_mulaw_table(int A, float* f32, short* i16_wrap, short* i16_saturate)
{
    if (A < 2) return fail(NVWN_EINVAL, "nvwn_mulaw_table: A must be at least 2");
    for (int x = 0; x < A; x++) {
        const double a = mulaw_expand(x, A);
        const long long iv = (long long)(32768.0 * a);                       // MAX_WAV_VALUE * audio, truncated (astype('int16'))
        if (f32) f32[x] = (float)a;
        if (i16_wrap) i16_wrap[x] = (short)(unsigned short)((unsigned long long)iv & 0xFFFFull);
        if (i16_saturate) i16_saturate[x] = (short)(iv > 32767 ? 32767 : (iv < -32768 ? -32768 : iv));
    }
    return 0;
}

int nvwn_get_audio(nvwn_engine* e, float* audio_f32, short* audio_i16, int offset, int size, int saturate, void* stream)
{
    if (!e || (!audio_f32 && !audio_i16)) return fail(NVWN_EINVAL, "nvwn_get_audio: NULL argument");
    if (offset < 0 || size < 0 || offset + size > e->N) return fail(NVWN_EINVAL, "nvwn_get_audio: range out of bounds");
    if (size == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    const int A = e->A;
    if (!e->lut_f) {
        // tables: float[A] | int16[A] (the reference's cast: trunc, code A-1 -> 32768 wraps to -32768) | int16[A] (clamped)
        std::vector<unsigned char> host((size_t)A * (sizeof(float) + 2 * sizeof(short)));
        float* hf = reinterpret_cast<float*>(host.data());
        short* hw = reinterpret_cast<short*>(host.data() + (size_t)A * sizeof(float));
        nvwn_mulaw_table(A, hf, hw, hw + A);
        CK(e->lut_f.alloc(host.size()));
        CK(cudaMemcpy(e->lut_f, host.data(), host.size(), cudaMemcpyHostToDevice));
    }
    const short* lut_s = reinterpret_cast<const short*>(e->lut_f + A) + (saturate ? A : 0);
    const size_t total = (size_t)e->B * size;
    const bool f_dev = !audio_f32 || is_device_ptr(audio_f32), s_dev = !audio_i16 || is_device_ptr(audio_i16);
    float* df = audio_f32;
    short* ds = audio_i16;
    DevBuf<char> tmp;
    if (!f_dev || !s_dev) {                                                   // host destination(s): decode into a device scratch, copy out
        CK(tmp.alloc(total * (sizeof(float) + sizeof(short))));
        if (!f_dev) df = reinterpret_cast<float*>(tmp.get());
        if (!s_dev) ds = reinterpret_cast<short*>(tmp + total * sizeof(float));
    }
    cudaError_t ce = wn_mulaw_decode(e->yOut, e->N, offset, size, e->B, A, e->lut_f, lut_s, df, ds, st);
    if (ce == cudaSuccess && !f_dev) ce = cudaMemcpyAsync(audio_f32, df, total * sizeof(float), cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess && !s_dev) ce = cudaMemcpyAsync(audio_i16, ds, total * sizeof(short), cudaMemcpyDeviceToHost, st);
    if (tmp && ce == cudaSuccess) ce = cudaStreamSynchronize(st);            // before tmp is freed on return
    if (ce != cudaSuccess) return fail((int)ce, std::string("nvwn_get_audio: ") + cudaGetErrorString(ce));
    return 0;
}

}  // extern "C"

namespace {

// The checks every scoring call shares, in their order: arguments, engine kind, batch_size.
int score_args(const nvwn_engine* e, const char* who, const int* audio, int batch_size, const float* logp)
{
    if (!e || !audio || !logp) return fail(NVWN_EINVAL, std::string(who) + ": NULL engine, audio or logp");
    if (e->dtype != NVWN_FP16) return fail(NVWN_EUNSUPPORTED, std::string(who) + ": only NVWN_FP16 engines can score");
    if (e->A != 256) return fail(NVWN_EUNSUPPORTED, std::string(who) + ": scoring needs A = 256");
    if (batch_size < 1 || batch_size > e->B) return fail(NVWN_EINVAL, std::string(who) + ": batch_size outside [1, B]");
    return 0;
}

// The checks of nvwn_score_stream (packed false) and nvwn_score_stream_packed, in their order: score_args, the starts flags, the window,
// and for a call that continues the open stream (first_sample != 0) its next sample, batch_size and kind.
int score_stream_args(const nvwn_engine* e, const std::string& who, const int* audio, const unsigned char* starts, bool packed, long long first_sample,
                      int count, int batch_size, const float* logp)
{
    int rc = score_args(e, who.c_str(), audio, batch_size, logp);
    if (rc == 0 && packed && !starts) rc = fail(NVWN_EINVAL, who + ": starts is NULL");
    if (rc == 0) rc = check_window(e, who, first_sample, count, "count", 1);
    if (rc != 0 || first_sample == 0) return rc;
    if (e->score_next < 0)
        return fail(NVWN_EINVAL, who + ": first_sample " + std::to_string(first_sample) + " continues no scoring stream (nvwn_score and weight "
                                       "changes end one): start one at first_sample = 0");
    if (first_sample != e->score_next)
        return fail(NVWN_EINVAL, who + ": first_sample " + std::to_string(first_sample) + " does not continue the scoring stream: the next sample is " +
                                     std::to_string(e->score_next) + " (first_sample = 0 starts over)");
    if (batch_size != e->score_bs)
        return fail(NVWN_EINVAL, who + ": batch_size " + std::to_string(batch_size) + " differs from the scoring stream's batch_size " +
                                     std::to_string(e->score_bs) + " (first_sample = 0 starts over)");
    if (packed != e->score_packed)
        return fail(NVWN_EINVAL, who + ": the scoring stream is " + (e->score_packed ? "packed: continue it with nvwn_score_stream_packed"
                                                                                    : "not packed: continue it with nvwn_score_stream") +
                                     " (first_sample = 0 starts over)");
    return 0;
}

// The chunk loop of every scoring call: absolute samples [first, first + count) of the first Bs utterances, 1 <= count <= N, sample t
// with the conditioning at store position t mod N; audio, logp and logits hold [Bs][count] (host or device).  first == 0 starts
// afresh (x_l[t - d] = 0 for t < d, codes 128 / 128); any other first continues from the layer fronts and codes the last call left.
// keep leaves the call's own fronts and codes there and opens the stream at first + count; otherwise the stream ends.  starts (host or
// device [Bs][count], or NULL) packs the call: each row's local time, carried from the last call and 0 at a flag and at first == 0,
// selects the packed kernels' masks, and the stream it keeps open is packed.  The caller has checked the arguments; the audio is
// checked here, before any state changes.
int score_range(nvwn_engine* e, const char* who, const int* audio, const unsigned char* starts, long long first, int count, int Bs, float* logp,
                float* logits, bool keep, cudaStream_t st)
{
    const int N = count, L = e->L, R = e->R, A = e->A;
    if (!e->score_scratch) {
        int T = SCORE_ROWS / e->B;
        if (T < 1) T = 1;
        if (T > e->N) T = e->N;
        CK(e->score_scratch.alloc(score_scratch_layout(e, T).bytes));
        e->score_T = T;
    }
    const int T = e->score_T;
    const ScoreScratch o = score_scratch_layout(e, T);
    char* sc = e->score_scratch;
    int* d_audio = reinterpret_cast<int*>(sc + o.audio);
    int* d_codes = reinterpret_cast<int*>(sc + o.codes);
    unsigned long long* d_bad = reinterpret_cast<unsigned long long*>(sc + o.bad);
    __half* xh = reinterpret_cast<__half*>(sc + o.xh);

    // the audio is outside input: range-check it on the device whatever memory it is in, and name the first offender
    const size_t n_audio = (size_t)Bs * N;
    CK(cudaMemcpyAsync(d_audio, audio, n_audio * sizeof(int), cudaMemcpyDefault, st));
    CK(cudaMemsetAsync(d_bad, 0xff, sizeof(unsigned long long), st));
    CK(wn_score_check_audio(d_audio, n_audio, A, d_bad, st));
    unsigned long long bad = 0;
    CK(cudaMemcpyAsync(&bad, d_bad, sizeof bad, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (bad != ~0ull) {
        int v = 0;
        CK(cudaMemcpy(&v, d_audio + bad, sizeof v, cudaMemcpyDeviceToHost));
        return fail(NVWN_EINVAL, std::string(who) + ": audio[" + std::to_string(bad / N) + "][" + std::to_string(first + (long long)(bad % N)) + "] = " +
                                     std::to_string(v) + " is outside [0, " + std::to_string(A) + ")");
    }
    e->score_next = -1;                      // reopened below once this call's state is complete
    WnParams p;
    fill_params(e, p, 0, 0, 0, N, Bs, 0);
    // model 0's image, which a call reads unless a row runs another model; then, if one does, the call's segments
    WnScoreSegs segs{};
    bool by_model = false;
    for (int b = 0; b < Bs && !by_model; b++) by_model = score_model(e, b) != 0;
    int rc = put_score_image(e, 0, p, st);
    if (rc == 0 && by_model) rc = score_segments(e, p, Bs, segs, st);
    if (rc != 0) return rc;
    const bool logp_dev = is_device_ptr(logp), logits_dev = logits && is_device_ptr(logits);
    if (first == 0) {
        for (int l = 0; l < L; l++)          // x_l[t - d] = 0 for t < d
            CK(cudaMemsetAsync(xh + wn_score_xh_offset(l, L, e->maxDil, T, e->B, R), 0,
                               (size_t)wn_score_dilation(l, e->maxDil) * Bs * R * sizeof(__half), st));
        CK(wn_fill_int(d_codes, 128, (size_t)Bs * 2, st));
        if (starts) CK(cudaMemsetAsync(sc + o.carry, 0, (size_t)Bs * sizeof(int), st));
    }
    WnScoreChunk c;
    c.L = L; c.R = R; c.S = e->S; c.A = A; c.maxDil = e->maxDil; c.tanhEmbed = e->tanhEmbed;
    c.Bs = Bs; c.Be = e->B; c.N = N; c.Tcap = T;
    c.image = e->models[0].score_image; c.embPrev = e->models[0].blob + e->o_embPrev; c.embCur = e->models[0].blob + e->o_embCur;
    c.audio = d_audio;
    c.codes = d_codes;
    float* lh = reinterpret_cast<float*>(sc + o.lh);
    c.lh = lh;
    c.xh = xh;
    c.xf = reinterpret_cast<float*>(sc + o.xf);
    c.H = reinterpret_cast<__half*>(sc + o.H);
    c.logp = logp_dev ? logp : reinterpret_cast<float*>(sc + o.logp);
    c.starts = nullptr;
    c.segs = by_model ? &segs : nullptr;
    c.segs_dev = by_model ? e->score_segs.get() : nullptr;
    if (starts) {
        CK(cudaMemcpyAsync(sc + o.starts, starts, n_audio, cudaMemcpyDefault, st));
        c.starts = reinterpret_cast<const unsigned char*>(sc + o.starts);
        c.tau = reinterpret_cast<int*>(sc + o.tau);
        c.tau_carry = reinterpret_cast<int*>(sc + o.carry);
    }
    float* lgt = reinterpret_cast<float*>(sc + o.lgt);
    for (int t0 = 0; t0 < N; t0 += T) {
        const int Tc = N - t0 < T ? N - t0 : T;
        // the chunk's conditioning, in two pieces where its samples wrap around the store
        for (const WrapPiece& w : split_at_wrap(first + t0, Tc, e->N))
            CK(e->family->readback(*e, lh + (size_t)w.off * L * e->B * 2 * R, e->Lh, w.pos, w.len, st));
        c.t0 = t0; c.T = Tc;
        c.logits = logits ? (logits_dev ? logits : lgt) : nullptr;
        c.logits_ld = logits_dev ? (long long)N * A : (long long)Tc * A;
        c.logits_t0 = logits_dev ? 0 : t0;
        CK(wn_score_chunk(c, st));
        if (logits && !logits_dev)
            CK(cudaMemcpy2DAsync(logits + (size_t)t0 * A, (size_t)N * A * sizeof(float), lgt, (size_t)Tc * A * sizeof(float),
                                 (size_t)Tc * A * sizeof(float), Bs, cudaMemcpyDeviceToHost, st));
        if (t0 + Tc < N || keep) {
            // carry the last d_l steps of every layer's input to the front of its buffer, in pieces that do not overlap; after the
            // last chunk these are the fronts of the stream's next call
            const size_t piece = (size_t)Tc * Bs;
            for (int l = 0; l < L; l++) {
                __half* buf = xh + wn_score_xh_offset(l, L, e->maxDil, T, e->B, R);
                const size_t hist = (size_t)wn_score_dilation(l, e->maxDil) * Bs;
                for (size_t done = 0; done < hist; done += piece) {
                    const size_t m = hist - done < piece ? hist - done : piece;
                    CK(cudaMemcpyAsync(buf + done * R, buf + (piece + done) * R, m * R * sizeof(__half), cudaMemcpyDeviceToDevice, st));
                }
            }
        }
    }
    if (keep) {
        CK(wn_score_carry_codes(d_codes, d_audio, N, N, Bs, st));
        e->score_next = first + N;
        e->score_bs = Bs;
        e->score_packed = starts != nullptr;
    }
    if (!logp_dev) CK(cudaMemcpyAsync(logp, c.logp, n_audio * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (!logp_dev || (logits && !logits_dev)) CK(cudaStreamSynchronize(st));
    return 0;
}

}  // namespace

extern "C" {

int nvwn_score(nvwn_engine* e, const int* audio, int num_samples, int batch_size, float* logp, float* logits, void* stream)
{
    int rc = score_args(e, "nvwn_score", audio, batch_size, logp);
    if (rc != 0) return rc;
    if (num_samples < 1 || num_samples > e->N) return fail(NVWN_EINVAL, "nvwn_score: num_samples outside [1, N]");
    return score_range(e, "nvwn_score", audio, nullptr, 0, num_samples, batch_size, logp, logits, false, (cudaStream_t)stream);
}

int nvwn_score_stream(nvwn_engine* e, const int* audio, long long first_sample, int count, int batch_size, float* logp, float* logits, void* stream)
{
    const std::string who = "nvwn_score_stream";
    const int rc = score_stream_args(e, who, audio, nullptr, false, first_sample, count, batch_size, logp);
    if (rc != 0) return rc;
    return score_range(e, who.c_str(), audio, nullptr, first_sample, count, batch_size, logp, logits, true, (cudaStream_t)stream);
}

int nvwn_score_stream_packed(nvwn_engine* e, const int* audio, const unsigned char* starts, long long first_sample, int count, int batch_size,
                             float* logp, float* logits, void* stream)
{
    const std::string who = "nvwn_score_stream_packed";
    const int rc = score_stream_args(e, who, audio, starts, true, first_sample, count, batch_size, logp);
    if (rc != 0) return rc;
    return score_range(e, who.c_str(), audio, starts, first_sample, count, batch_size, logp, logits, true, (cudaStream_t)stream);
}

int nvwn_prime_from_score(nvwn_engine* e, void* stream)
{
    const std::string who = "nvwn_prime_from_score";
    int rc = check_open_stream(e, who, "history to generate from");
    if (rc == 0) rc = check_run_batch(e, who, e->score_bs);
    if (rc == 0) rc = check_prime_model(e, who, nullptr, nullptr, e->score_bs);
    if (rc != 0) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int Bs = e->score_bs;
    rc = put_fronts(e, [&](int l, const __half* src, long long t_first, int n_t) {
        return e->family->put_history(*e, e->ring, src, l, t_first, n_t, Bs, st);
    });
    if (rc != 0) return rc;
    CK(wn_feedback_from_codes(reinterpret_cast<const int*>(e->score_scratch + score_scratch_layout(e, e->score_T).codes), Bs, e->yPrev, e->yCur, st));
    e->next_t = e->score_next;
    e->prime_bs = Bs;
    return 0;
}

int nvwn_prime_slots_from_score(nvwn_engine* e, const int* rows, const int* slots, int n, const unsigned long long* seeds, void* stream)
{
    const std::string who = "nvwn_prime_slots_from_score";
    int rc = check_open_stream(e, who, "history to generate from");
    if (rc != 0) return rc;
    if (!rows) return fail(NVWN_EINVAL, who + ": rows is NULL");
    if ((rc = check_slots(e, who, slots, n)) || (rc = check_rows(e, who, rows, n)) || (rc = check_prime_model(e, who, rows, slots, n))) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned long long* seeds_dev;
    if ((rc = take_slots(e, who, slots, n, seeds, &seeds_dev, st)) || (rc = copy_snapshot(e->prime_rows, rows, n, st)) || (rc = clear_early_times(e, st)))
        return rc;
    const int Bs = e->score_bs;
    const long long P = e->score_next, origin = e->next_t - P;
    // what nvwn_restart_slots at origin = next_t - P does to these slots, then nvwn_prime_from_score of their rows with local time tau
    // at engine time origin + tau
    CK(e->family->clear_rows(*e, e->ring, e->slot_rows, n, st));
    rc = put_fronts(e, [&](int l, const __half* src, long long tau, int n_t) {
        return e->family->put_history_rows(*e, e->ring, src, e->prime_rows, e->R, (size_t)Bs * e->R, e->slot_rows, n, l, origin + tau, n_t, st);
    });
    if (rc != 0) return rc;
    CK(wn_prime_rows(reinterpret_cast<const int*>(e->score_scratch + score_scratch_layout(e, e->score_T).codes), e->prime_rows, e->slot_rows, n, seeds_dev,
                     origin, e->yPrev, e->yCur, e->origin, e->seed, st));
    return 0;
}

int nvwn_slot_state_bytes(nvwn_engine* e, unsigned long long* bytes)
{
    if (!e || !bytes) return fail(NVWN_EINVAL, "nvwn_slot_state_bytes: NULL argument");
    *bytes = wn_slot_state_bytes(*e);
    return 0;
}

int nvwn_save_slots(nvwn_engine* e, const int* slots, int n, void* states, void* stream)
{
    const std::string who = "nvwn_save_slots";
    if (!e || !states) return fail(NVWN_EINVAL, who + ": NULL argument");
    const int rc = check_slots(e, who, slots, n);
    if (rc != 0) return rc;
    const size_t bytes = wn_slot_state_bytes(*e);
    cudaStream_t st = (cudaStream_t)stream;
    return write_states(e, who, states, n, st, [&](char* dst) {
        // the slot list goes through the slot scratch, but this is no per-slot call: the engine does not change
        const int rc = copy_snapshot(e->slot_rows, slots, n, st);
        if (rc != 0) return rc;
        CK(wn_save_slot_scalars(dst, bytes, e->slot_rows, n, *e, e->next_t, e->yPrev, e->yCur, e->origin, e->seed, st));
        return state_layers(e, [&](int l, size_t off, int d) {
            return e->family->get_history_rows(*e, e->ring, dst + off, bytes / e->td, e->R, e->slot_rows, n, l, e->next_t - d, d, e->origin, st);
        });
    });
}

int nvwn_score_save_states(nvwn_engine* e, const int* rows, int n, const unsigned long long* seeds, void* states, void* stream)
{
    const std::string who = "nvwn_score_save_states";
    int rc = check_open_stream(e, who, "utterance's state");
    if (rc != 0) return rc;
    if (!rows || !states) return fail(NVWN_EINVAL, who + ": NULL argument");
    const int Bs = e->score_bs;
    if (n < 1 || n > Bs) return fail(NVWN_EINVAL, who + ": n " + std::to_string(n) + " is outside [1, " + std::to_string(Bs) + "] (the scoring stream's batch_size)");
    if ((rc = check_rows(e, who, rows, n))) return rc;
    const size_t bytes = wn_slot_state_bytes(*e);
    cudaStream_t st = (cudaStream_t)stream;
    return write_states(e, who, states, n, st, [&](char* dst) {
        // rows and seeds go through the per-call scratch of the primes; nothing else of the engine is touched
        int rc;
        if ((rc = copy_snapshot(e->prime_rows, rows, n, st)) || (seeds && (rc = copy_snapshot(e->slot_seeds, seeds, n, st)))) return rc;
        const ScoreScratch o = score_scratch_layout(e, e->score_T);
        CK(wn_score_save_states(dst, bytes, reinterpret_cast<const __half*>(e->score_scratch + o.xh), reinterpret_cast<const int*>(e->score_scratch + o.codes),
                                e->prime_rows, n, seeds ? e->slot_seeds.get() : nullptr, *e, e->score_next, e->score_T, e->B, Bs, st));
        return 0;
    });
}

int nvwn_load_slots(nvwn_engine* e, const int* slots, int n, const void* states, void* stream)
{
    const std::string who = "nvwn_load_slots";
    if (!e || !states) return fail(NVWN_EINVAL, who + ": NULL argument");
    int rc = check_slots(e, who, slots, n);
    if (rc != 0) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    bool host;
    if ((rc = check_states(who, states, &host))) return rc;
    const size_t bytes = wn_slot_state_bytes(*e), hb = sizeof(nvwn_slot_state_header);
    // every header is checked before anything changes; device headers are read in stream order (the call runs at a window boundary)
    std::vector<nvwn_slot_state_header> h(n);
    if (host) {
        for (int i = 0; i < n; i++) memcpy(&h[i], static_cast<const char*>(states) + (size_t)i * bytes, hb);
    } else {
        CK(cudaMemcpy2DAsync(h.data(), hb, states, bytes, hb, n, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
    }
    for (int i = 0; i < n; i++) {
        const nvwn_slot_state_header& x = h[i];
        const std::string s = "state " + std::to_string(i);
        if (x.tag != NVWN_SLOT_STATE_TAG) return fail(NVWN_EINVAL, who + ": " + s + " is not a slot state (nvwn_save_slots)");
        if (x.dtype != e->dtype || x.R != e->R || x.L != e->L || x.max_dilation != e->maxDil)
            return fail(NVWN_EINVAL, who + ": " + s + " has dtype " + std::to_string(x.dtype) + ", R " + std::to_string(x.R) + ", L " + std::to_string(x.L) +
                                         " and max_dilation " + std::to_string(x.max_dilation) + "; the engine has " + std::to_string(e->dtype) + ", " +
                                         std::to_string(e->R) + ", " + std::to_string(e->L) + " and " + std::to_string(e->maxDil));
        if (x.position < 0 || x.y_prev < 0 || x.y_prev >= e->A || x.y_cur < 0 || x.y_cur >= e->A)
            return fail(NVWN_EINVAL, who + ": " + s + " has position " + std::to_string(x.position) + " and fed-back indices " + std::to_string(x.y_prev) +
                                         ", " + std::to_string(x.y_cur) + "; need position >= 0 and indices in [0, " + std::to_string(e->A) + ")");
    }
    const char* src = static_cast<const char*>(states);
    if (host) {
        CK(e->state_stage.reserve((size_t)n * bytes));
        if ((rc = copy_snapshot(e->state_stage, src, (size_t)n * bytes, st))) return rc;
        src = e->state_stage;
    }
    if ((rc = take_slots(e, who, slots, n, nullptr, nullptr, st)) || (rc = clear_early_times(e, st))) return rc;
    const long long t0 = e->next_t;
    CK(e->family->clear_rows(*e, e->ring, e->slot_rows, n, st));
    rc = state_layers(e, [&](int l, size_t off, int d) {
        return e->family->put_history_rows(*e, e->ring, src + off, nullptr, bytes / e->td, e->R, e->slot_rows, n, l, t0 - d, d, st);
    });
    if (rc != 0) return rc;
    CK(wn_load_slot_scalars(src, bytes, e->slot_rows, n, t0, e->yPrev, e->yCur, e->origin, e->seed, st));
    return 0;
}

// debug only (not part of the public ABI): the engine's conditioning store for samples [first_sample, first_sample + num_samples),
// converted back to fp32 [num_samples][L][B][2R] whatever the kernel-native layout (plain / tiled fp16 / fragment order) is
int nvwn_debug_get_conditioning(nvwn_engine* e, float* out, int first_sample, int num_samples)
{
    if (!e || !out) return fail(NVWN_EINVAL, "nvwn_debug_get_conditioning: NULL argument");
    if (first_sample < 0 || num_samples < 0 || first_sample + num_samples > e->N) return fail(NVWN_EINVAL, "nvwn_debug_get_conditioning: range out of bounds");
    const size_t per = (size_t)e->L * e->B * 2 * e->R, n = per * num_samples;
    if (n == 0) return 0;
    DevBuf<float> tmp;
    CK(tmp.alloc(n * sizeof(float)));
    cudaError_t ce = e->family->readback(*e, tmp, e->Lh, first_sample, num_samples, 0);
    if (ce == cudaSuccess) ce = cudaMemcpy(out, tmp, n * sizeof(float), cudaMemcpyDefault);
    if (ce != cudaSuccess) return fail((int)ce, std::string("nvwn_debug_get_conditioning: ") + cudaGetErrorString(ce));
    return 0;
}

// debug only (not part of the public ABI): the whole history ring, read at the stride of a run of `batch` utterances, as fp32
// [(maxDil+1)][L][batch][R] in slot order, whatever the kernel-native layout
int nvwn_debug_get_history(nvwn_engine* e, float* out, int batch)
{
    if (!e || !out) return fail(NVWN_EINVAL, "nvwn_debug_get_history: NULL argument");
    if (batch < 1 || batch > e->B) return fail(NVWN_EINVAL, "nvwn_debug_get_history: batch outside [1, B]");
    const size_t n = (size_t)(e->maxDil + 1) * e->L * batch * e->R;
    DevBuf<float> tmp;
    CK(tmp.alloc(n * sizeof(float)));
    cudaError_t ce = e->family->get_history(*e, tmp, e->ring, batch, nullptr, 0);
    if (ce == cudaSuccess) ce = cudaMemcpy(out, tmp, n * sizeof(float), cudaMemcpyDefault);
    if (ce != cudaSuccess) return fail((int)ce, std::string("nvwn_debug_get_history: ") + cudaGetErrorString(ce));
    return 0;
}

// debug only (not part of the public ABI): rows rows[0..n) (host memory; distinct, in [0, B)) of every history-ring entry, as fp32
// [(maxDil+1)][L][n][R] in slot order: what nvwn_debug_get_history reads for those rows, without reading back a whole large ring
int nvwn_debug_get_history_rows(nvwn_engine* e, float* out, const int* rows, int n)
{
    if (!e || !out) return fail(NVWN_EINVAL, "nvwn_debug_get_history_rows: NULL argument");
    int rc = check_slots(e, "nvwn_debug_get_history_rows", rows, n);
    if (rc != 0) return rc;
    const size_t count = (size_t)(e->maxDil + 1) * e->L * n * e->R;
    DevBuf<int> rows_dev;
    DevBuf<float> tmp;
    CK(rows_dev.alloc(n * sizeof(int)));
    CK(tmp.alloc(count * sizeof(float)));
    cudaError_t ce = cudaMemcpy(rows_dev, rows, n * sizeof(int), cudaMemcpyHostToDevice);
    if (ce == cudaSuccess) ce = e->family->get_history(*e, tmp, e->ring, n, rows_dev, 0);
    if (ce == cudaSuccess) ce = cudaMemcpy(out, tmp, count * sizeof(float), cudaMemcpyDefault);
    if (ce != cudaSuccess) return fail((int)ce, std::string("nvwn_debug_get_history_rows: ") + cudaGetErrorString(ce));
    return 0;
}

// debug only (not part of the public ABI): record a clock64 timeline of sample `t` of block 0 into `out` (3 x 1024 words)
int nvwn_debug_trace(nvwn_engine* e, int t, unsigned long long* out_host, int fetch)
{
    if (!e) return NVWN_EINVAL;
    if (!fetch) {
        if (!e->trace) CK(e->trace.alloc(3 * 1024 * sizeof(unsigned long long)));
        CK(cudaMemset(e->trace, 0, 3 * 1024 * sizeof(unsigned long long)));
        e->trace_t = t;
        return 0;
    }
    CK(cudaMemcpy(out_host, e->trace, 3 * 1024 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return 0;
}

// debug only: how many three-CTA clusters of `rows` (8 or 16) utterances the latency kernel runs at once (batches up to rows x this
// can use that tile height)
int nvwn_debug_lat_max_clusters(int S, int rows) { return wn_lat_max_clusters(S, rows); }

int nvwn_get_launch_info(nvwn_engine* e, nvwn_launch_info* info)
{
    if (!e || !info) return fail(NVWN_EINVAL, "nvwn_get_launch_info: NULL argument");
    info->kernel = e->last.kernel; info->grid = e->last.grid; info->block = e->last.block;
    info->smem_bytes = e->last.smem_bytes; info->batch_per_cta = e->last.batch_per_cta; info->cluster = e->last.cluster;
    info->launches = e->launches;
    const unsigned long long R = e->R, S = e->S, A = e->A, L = e->L;
    info->weight_bytes = e->td * (L * (2 * 2 * R * R + R * R + S * R + 3 * R + S) + A * S + A * A + 2 * A);
    return 0;
}

}  // extern "C"
