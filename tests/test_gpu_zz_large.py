"""Large batches and deep histories on the fp16 kernels.

The history ring holds (maxDil + 1) x L entries, one per (slot, layer), each with every utterance's layer input of one sample.
At large batches and deep stacks it passes 4 GiB, and every byte offset into it has to be formed in 64 bits: an offset that wraps
at 2^32 still lies inside the allocation, so nothing faults and the kernel silently reads and writes another entry's bytes.

test_ring_past_4gib runs a ring just past 4 GiB on each latency kernel (8-row clusters, 16-row clusters, the single-CTA kernel)
and, as controls, on the tensor-core and fp16 stream kernels: a streaming engine with a small window runs past the first entry
whose offset reaches 2^32, and rows at both ends of the batch must equal, bit for bit, an engine of only those rows -- the
samples, the last step's dumps and the history the rows hold.  Rows are independent and every tile height gives the same bits
(test_gpu_lat_tile_height.py), so any difference is an addressing error; the history comparison sees the first wrapped write
before any sample is drawn from it.  The last rows are then saved, loaded into a fresh engine and continued: equal to the run
that went on uninterrupted.  test_ring_configurations_pass_4gib (no GPU) keeps those configurations past 4 GiB.

test_auto_regimes_at_c3 runs C3 with nothing forced at each batch regime AUTO picks: the largest batch of resident 8-row
clusters and one more utterance, the largest of resident 16-row clusters and one more (the single-CTA kernel), and 2 560
utterances (the single-CTA kernel in two waves).  Rows at cluster, tile and wave edges equal a small single-CTA engine of those
rows bit for bit, and four of them, replayed through the fp32 oracle as its forced history, have every sampled index in its
window of the oracle's distribution (tests/replay.py).

Every large engine is created alone and closed before the next, and a case skips when the shared device has too little memory
free.  On an H100 80GB HBM3 (700 W) the file ran in about 30 s, with at most 6.8 GiB of device memory in use (lat_single).
"""
import ctypes as C

import numpy as np
import pytest

import nv_wavenet_b200 as nw
from nv_wavenet_b200 import _lib
from tests import refgen, replay
from tests.common import bits_equal

R, S, A = 64, 256, 256
W = 32                                   # window of every streaming engine: the conditioning store stays small
TU, TC_TILE, TC_TILE_BYTES = 16, 64, 16384
ENV_KEYS = ("NVWN_FP16_KERNEL", "NVWN_LAT_CLUSTER", "NVWN_LAT_MAX_B", "NVWN_TC_TILE", "NVWN_TC_NODUP", "NVWN_TC_FUSED",
            "NVWN_STREAM_BT", "NVWN_STREAM_RING")
LAT = {"NVWN_FP16_KERNEL": "lat"}
LAT_SINGLE = {"NVWN_FP16_KERNEL": "lat", "NVWN_LAT_CLUSTER": "0"}
TC = {"NVWN_FP16_KERNEL": "tc"}
STREAM = {"NVWN_FP16_KERNEL": "stream", "NVWN_STREAM_BT": "4"}     # 4 rows per CTA at every batch of the case: the same arithmetic

# case -> (L, maxDil, B, steps before the save, family, environment, launch info it must report); the reference engines of a case
# run the single-CTA latency kernel (latency cases) or the case's own environment (controls)
RING_CASES = {
    "lat_8row": (64, 2048, 256, 2080, "lat", LAT, {"kernel": 18, "cluster": 3, "batch_per_cta": 8}),
    "lat_16row": (41, 2048, 400, 2080, "lat", LAT, {"kernel": 18, "cluster": 3, "batch_per_cta": 16}),
    "lat_single": (20, 512, 3265, 544, "lat", LAT_SINGLE, {"kernel": 18, "cluster": 1, "batch_per_cta": 16}),
    "tc": (64, 2048, 128, 2080, "tc", TC, {"kernel": 17}),
    "stream_fp16": (64, 2048, 256, 2080, "stream", STREAM, {"kernel": 16, "batch_per_cta": 4}),
}


def ring_layout(family, L, md, B):
    """(ring bytes, bytes per ring entry) of an fp16 engine of `family`: LatLayout, TcLayout (64-row tiles) or PlainLayout."""
    if family == "lat":
        entry = -(-B // TU) * 2048
    elif family == "tc":
        entry = -(-B // TC_TILE) * TC_TILE_BYTES
    else:
        entry = B * R * 2
    return (md + 1) * L * entry, entry


def first_entry_past_4gib(family, L, md, B):
    """(slot, layer) of the first ring entry whose byte offset is 2^32 or more, or None."""
    ring, entry = ring_layout(family, L, md, B)
    e = -(-(1 << 32) // entry)
    return divmod(e, L) if e < (md + 1) * L else None


def test_ring_configurations_pass_4gib():
    """Each case's ring is past 4 GiB -- so the latency kernels run their 64-bit-offset instantiations -- and its run writes the
    first entry at or past 2^32 at least W steps before the save, so the comparisons read what a wrapped offset would have
    corrupted.  (The latency cases need L <= 64.)"""
    want_first = {"lat_8row": (2048, 0), "lat_16row": (2046, 1), "lat_single": (511, 11), "tc": (2048, 0), "stream_fp16": (2048, 0)}
    for case, (L, md, B, T, family, _, _) in RING_CASES.items():
        ring, entry = ring_layout(family, L, md, B)
        assert (1 << 32) < ring < (1 << 32) * 1.01, (case, ring)
        first = first_entry_past_4gib(family, L, md, B)
        assert first == want_first[case], (case, first)
        slot, _ = first
        assert slot + W <= T and T % W == 0 and L <= 64, case         # slot = the sample that writes it (the run starts at 0)
    # the single-CTA case is the smallest C3 batch past 4 GiB
    assert ring_layout("lat", 20, 512, 3265 - 1)[0] < (1 << 32) < ring_layout("lat", 20, 512, 3265)[0]


# ------------------------------------------------------------------------------------------------ helpers (GPU)
def _engine(env, L, md, B, monkeypatch):
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    return nw.NVWavenetInfer(L, md, B, W, R=R, S=S, A=A, dtype=nw.FP16)


def _weights(seed, L):
    """lively weights with a peaked output layer (the c3 configuration of test_gpu_zz_replay.py)"""
    w = refgen.lively_inputs(seed, R, S, A, L, 1, 1)
    w["Wza"] = (w["Wza"] * np.float32(5.0)).astype(np.float32)
    return w


def _window(seed, first, L, B):
    """Conditioning [W][L][B][2R] (N(0, 0.5^2), as refgen.lively_inputs draws it) and selectors [W][B] of samples [first, first + W)
    of a B-utterance batch, drawn on the device: an engine serving some of its rows is given those rows."""
    import torch
    g = torch.Generator(device="cuda")
    g.manual_seed(seed * 1000003 + first)
    lh = torch.randn((W, L, B, 2 * R), generator=g, device="cuda").mul_(0.5)
    return lh, torch.rand((W, B), generator=g, device="cuda")


class _Rows:
    """A streaming engine serving rows `rows` of the batch (None: all), its sample 0 at the batch's sample t0; y [rows][samples]."""

    def __init__(self, e, w, rows=None, t0=0):
        self.e, self.rows, self.t0, self.y = e, rows, t0, []
        e.load(w)
        e.reset_history()

    def run(self, lh, sel, first, dump):
        t = first - self.t0
        if self.rows is not None:
            lh, sel = lh[:, :, self.rows].contiguous(), sel[:, self.rows].contiguous()
        self.e.set_conditioning_stream(lh, t)
        self.e.set_selectors(sel)                              # positions t mod W: every window starts at a multiple of W
        self.e.run_stream(t, W, self.e.B, dump_activations=dump)
        y = np.empty((self.e.B, W), np.int32)
        self.e.get_yout_stream(y, t, W)
        self.y.append(y)

    def samples(self):
        return np.concatenate(self.y, axis=1)


def _drive(engines, seed, L, B, first, last, keep=None):
    """Windows [first, last) of the batch through every engine, dumping the last step; keep(lh, sel) sees each window."""
    for f in range(first, last, W):
        lh, sel = _window(seed, f, L, B)
        for r in engines:
            r.run(lh, sel, f, f + W == last)
        if keep:
            keep(lh, sel)


def _history(e, rows):
    """rows `rows` of every history-ring entry of engine e, fp32 [(maxDil+1)][L][len(rows)][R]"""
    lib = _lib.lib()
    lib.nvwn_debug_get_history_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    r = np.ascontiguousarray(rows, dtype=np.int32)
    out = np.full((e.max_dilation + 1, e.L, r.size, R), np.nan, np.float32)
    assert lib.nvwn_debug_get_history_rows(e._h, C.c_void_p(out.ctypes.data), C.c_void_p(r.ctypes.data), r.size) == 0
    return out


def _dumps(e, rows=None):
    a = e.activations()
    pick = slice(None) if rows is None else list(rows)
    return {"xt": a["xt"][:, pick], "skip": a["skip"][:, pick], "zs": a["zs"][pick], "za": a["za"][pick], "p": a["p"][pick]}


def _assert_rows_equal(big, rows, small, what, history=True):
    """rows `rows` of engine run `big` against every row of `small`: (history) the ring, which names the first misplaced entry,
    then the samples and the last step's dumps"""
    if history:
        hb, hs = _history(big.e, rows), _history(small.e, range(small.e.B))
        diff = np.argwhere(hb.view(np.uint32) != hs.view(np.uint32))
        assert diff.size == 0, f"{what}: {len(diff)} history values differ; first (slot, layer, row) {tuple(diff[0][:3])}"
    yb, ys = big.samples()[rows], small.samples()
    t = yb.shape[1] - ys.shape[1]                              # small started at big's sample t
    bad = np.argwhere(yb[:, t:] != ys)
    assert bad.size == 0, f"{what}: {len(bad)} samples differ; first (row {rows[bad[0][0]]}, sample {t + bad[0][1]})"
    db, ds = _dumps(big.e, rows), _dumps(small.e)
    for k in db:
        assert bits_equal(db[k], ds[k]), f"{what}: last-step dump {k} differs"


def _free_or_skip(need, what):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"{what}: needs {need / 2**30:.1f} GiB of device memory, {free / 2**30:.1f} GiB free on this shared device")
    return free


def _need(family, L, md, B):
    """device bytes a case needs, at most: the ring, twice an fp32 window (the window itself and the conditioning store), and 1 GiB
    for the rest (dumps, the reference engines, the history read back)"""
    ring, _ = ring_layout(family, L, md, B)
    return ring + 2 * W * L * -(-B // TU) * TU * 2 * R * 4 + (1 << 30)


def _fits():
    return tuple(_lib.lib().nvwn_debug_lat_max_clusters(S, rows) for rows in (8, 16))


def _edge_rows(B, extra=()):
    """first and last rows of the batch, 8- and 16-row tile edges at both ends, and `extra` (sorted, distinct, at most 16)"""
    rows = {0, 7, 8, 15, 16, B - 17, B - 16, B - 9, B - 8, B - 1} | set(extra)
    rows = sorted(r for r in rows if 0 <= r < B)
    assert len(rows) <= TU
    return rows


# ------------------------------------------------------------------------------------------------ rings past 4 GiB
@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(RING_CASES))
def test_ring_past_4gib(case, monkeypatch):
    import torch
    L, md, B, T, family, env, want = RING_CASES[case]
    fit8, fit16 = _fits()
    if case == "lat_8row" and -(-B // 8) > fit8:
        pytest.skip(f"{fit8} resident 8-row clusters: {B} utterances do not run on 8-row clusters on this device")
    if case == "lat_16row" and not (-(-B // 8) > fit8 and -(-B // TU) <= fit16):
        pytest.skip(f"{fit8} / {fit16} resident 8- / 16-row clusters: {B} utterances do not run on 16-row clusters on this device")
    ref_env = LAT_SINGLE if family == "lat" else env
    rows = _edge_rows(B, (B // 2 - 1, B // 2))
    last = [B - 4, B - 3, B - 2, B - 1]                          # saved after the wrap and resumed in a fresh engine
    seed = 1000 + L
    w = _weights(seed, L)
    torch.cuda.empty_cache()
    free0 = _free_or_skip(_need(family, L, md, B), case)

    big = _Rows(_engine(env, L, md, B, monkeypatch), w)
    small = _Rows(_engine(ref_env, L, md, len(rows), monkeypatch), w, rows)
    _drive([big, small], seed, L, B, 0, T)
    torch.cuda.synchronize()
    used = free0 - torch.cuda.mem_get_info()[0]
    info = big.e.launch_info()
    assert all(info[k] == v for k, v in want.items()), info
    assert len(np.unique(big.samples()[rows])) > 32
    _assert_rows_equal(big, rows, small, f"{case}, {T} samples")

    states = big.e.save_slots(last)
    resumed = _Rows(_engine(ref_env, L, md, len(last), monkeypatch), w, last, t0=T)
    resumed.e.load_slots(list(range(len(last))), states)
    _drive([big, small, resumed], seed, L, B, T, T + W)
    _assert_rows_equal(big, rows, small, f"{case}, {T + W} samples")
    _assert_rows_equal(big, last, resumed, f"{case}, resumed at {T}", history=False)
    print(f"{case}: ring {ring_layout(family, L, md, B)[0] / 2**30:.3f} GiB, first entry past 4 GiB at (slot, layer) "
          f"{first_entry_past_4gib(family, L, md, B)}, {T + W} samples, {used / 2**30:.2f} GiB of device memory in use, {info}")
    for r in (big, small, resumed):
        r.e.close()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ every AUTO regime at C3
C3 = (20, 512)
T_C3 = 544                                                       # the 513-slot ring turns once
REGIMES = ["8row_full", "8row_plus1", "16row_full", "16row_plus1", "two_waves"]


def _regime_batch(regime, fit8, fit16):
    return {"8row_full": 8 * fit8, "8row_plus1": 8 * fit8 + 1, "16row_full": TU * fit16, "16row_plus1": TU * fit16 + 1,
            "two_waves": 2560}[regime]


def _auto_rows_per_cluster(B, fit8, fit16):
    """the engine's rule (lat_cluster_rows): 8-row clusters while all are resident, else 16-row ones, else the single-CTA kernel (0)"""
    return 8 if -(-B // 8) <= fit8 else TU if -(-B // TU) <= fit16 else 0


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES)
def test_auto_regimes_at_c3(regime, monkeypatch):
    import torch
    L, md = C3
    fit8, fit16 = _fits()
    if not fit8 or not fit16:
        pytest.skip("the device runs no three-CTA cluster of the latency kernel")
    B = _regime_batch(regime, fit8, fit16)
    tr = _auto_rows_per_cluster(B, fit8, fit16)
    want_tr = {"8row_full": 8, "8row_plus1": TU, "16row_full": TU, "16row_plus1": 0, "two_waves": 0}[regime]
    if tr != want_tr:
        pytest.skip(f"{fit8} / {fit16} resident 8- / 16-row clusters: {B} utterances are not in the {regime} regime on this device")
    prop = torch.cuda.get_device_properties(0)
    wave = TU * prop.multi_processor_count                       # rows of one wave of the single-CTA kernel at one CTA per SM
    rows = _edge_rows(B, (wave - 1, wave) if wave < B else (B // 2 - 1, B // 2))
    followed = [0, wave if wave < B else 15, B - 8, B - 1]       # replayed through the oracle
    seed = 2000 + B
    w = _weights(seed, L)
    torch.cuda.empty_cache()
    _free_or_skip(_need("lat", L, md, B), regime)

    big = _Rows(_engine({}, L, md, B, monkeypatch), w)
    small = _Rows(_engine(LAT_SINGLE, L, md, len(rows), monkeypatch), w, rows)
    lh_f, sel_f = [], []
    _drive([big, small], seed, L, B, 0, T_C3,
           keep=lambda lh, sel: (lh_f.append(lh[:, :, followed].cpu().numpy()), sel_f.append(sel[:, followed].cpu().numpy())))
    torch.cuda.synchronize()

    info = big.e.launch_info()
    assert info["kernel"] == 18 and info["batch_per_cta"] == (tr or TU), info
    if tr:
        assert info["cluster"] == 3 and info["grid"] == 3 * -(-B // tr), info
    else:
        assert info["cluster"] == 1 and info["grid"] == -(-B // TU), info
        per_sm = prop.shared_memory_per_multiprocessor // (info["smem_bytes"] + 1024)
        waves = -(-info["grid"] // (per_sm * prop.multi_processor_count))
        assert waves == (2 if regime == "two_waves" else 1), (info, per_sm)
    assert small.e.launch_info()["cluster"] == 1
    _assert_rows_equal(big, rows, small, f"C3 B = {B} ({regime})")

    y = np.ascontiguousarray(big.samples()[followed])
    assert len(np.unique(y)) > 32
    v = dict(w)
    v["Lh"], v["selectors"] = np.concatenate(lh_f), np.concatenate(sel_f)
    _, logits = replay.oracle_trace(v, range(len(followed)), (R, S, A, L, md), T_C3, forced=y)
    amb = replay.check(y, logits, v["selectors"], replay.DELTA, replay.MAX_AMBIGUOUS, what=f"C3 B = {B} ({regime}) rows {followed}: ")
    print(f"{regime}: B = {B}, {info}, rows {rows}, replayed {followed}: ambiguous {amb:.3f}")
    big.e.close(); small.e.close()
    torch.cuda.empty_cache()
