"""Every sampled index of the fp16 generation kernels against the CPU oracle's distribution (tests/replay.py).

The other fp16 tests compare logits at a few steps, or one launch split against another.  Here every step of long launches
without dumps -- the instantiation bench and serving run -- is replayed through the fp32 oracle, on every fp16 kernel variant
and FP32_FAST, in two configurations:

  export  the configuration a PyTorch model's export_weights() gives (refgen.export_inputs): no embedding tanh, zero embPrev,
          no output biases, a zero last residual layer; L16 maxDil 128, so the 129-slot history ring wraps 9 times in 1200 steps
  c3      lively weights with a peaked output layer, L20 maxDil 512: the ring wraps twice

Batches are 20 utterances on the latency and stream kernels (ragged 8- and 16-row tiles) and 130 on the tensor-core ones
(64- and 128-row tiles, the last nearly empty); the oracle follows the rows at tile edges (ROWS).  One oracle trace per
configuration serves every kernel and launch shape forced with its history.

delta (replay.DELTA, 6e-3) is the CDF distance from a boundary inside which a selector may fall either way; the fraction of
steps whose window then holds more than one class is bounded by replay.MAX_AMBIGUOUS (0.35).  Measured on an H100 SXM (80 GB HBM3, 700 W)
at the logit dumps of test_logits_where_ring_reads_change, the largest |CDF_kernel - CDF_fp32| was 2.1e-3 (the latency
kernels on c3; 1.4e-3 to 1.8e-3 on the others, 2e-6 for FP32_FAST), and that test keeps it below delta / 2.  The ambiguous
fraction was 0.20-0.21 on export and 0.14-0.15 on c3."""
import numpy as np
import pytest

import nv_wavenet_b200 as nw
from oracle import pyoracle as po
from tests import refgen, replay
from tests.test_gpu_parity import FP16_KERNELS, _logit_check, _select_fp16_kernel, gpu_engine
from tests.test_gpu_zz_selectors import philox_selectors

pytestmark = pytest.mark.gpu

R, S, A = 64, 256, 256
# name -> (L, maxDil, N, tanh_embed, delta, max ambiguous fraction)
CONFIGS = {
    "export": (16, 128, 1200, False, replay.DELTA, replay.MAX_AMBIGUOUS),
    "c3": (20, 512, 1200, True, replay.DELTA, replay.MAX_AMBIGUOUS),
}
B_LAT, B_TC = 20, 130
ROWS = [0, 7, 8, 15, 16, 19, 31, 32, 63, 64, 127, 128, 129]      # first/last of 8-row clusters, g and g+8, 64-row tile edges, ragged last rows
FP16_ROWS = [7, 8, 19, 129]                                     # rows the PREC_FP16 oracle follows, on a short prefix
FP16_PREFIX = 130
VARIANTS = FP16_KERNELS + ["fp32_fast"]
WINDOW = 100                                                    # divides neither 129 nor 513


def _inputs(name):
    L, md, N, tanh_embed = CONFIGS[name][:4]
    if name == "export":
        return refgen.export_inputs(90, R, S, A, L, B_TC, N)
    w = refgen.lively_inputs(91, R, S, A, L, B_TC, N)
    w["Wza"] = (w["Wza"] * np.float32(5.0)).astype(np.float32)
    return w


@pytest.fixture(scope="module")
def traces():
    """name -> (inputs of B_TC utterances, the fp32 oracle's free-running trajectory of ROWS, its logits [ROWS][N][A], and the
    PREC_FP16 oracle's logits [FP16_ROWS][FP16_PREFIX][A] under that history)."""
    out = {}

    def get(name):
        if name not in out:
            L, md, N, tanh_embed = CONFIGS[name][:4]
            w = _inputs(name)
            y, z = replay.oracle_trace(w, ROWS, (R, S, A, L, md), N, tanh_embed=tanh_embed)
            assert len(np.unique(y)) > 32
            fr = [ROWS.index(r) for r in FP16_ROWS]
            _, z16 = replay.oracle_trace(w, FP16_ROWS, (R, S, A, L, md), FP16_PREFIX, forced=y[fr], tanh_embed=tanh_embed,
                                         prec=po.PREC_FP16)
            out[name] = (w, y, z, z16)
        return out[name]
    return get


def _batch(variant):
    return B_TC if variant.startswith("tc") else B_LAT


def _engine(variant, w, L, B, N, md, tanh_embed, monkeypatch):
    _select_fp16_kernel("stream" if variant == "fp32_fast" else variant, monkeypatch)     # FP32_FAST ignores the fp16 switches
    dtype = nw.FP32_FAST if variant == "fp32_fast" else nw.FP16
    v = replay.sub_rows(w, range(B))
    v["Lh"] = np.ascontiguousarray(v["Lh"][:N]); v["selectors"] = np.ascontiguousarray(v["selectors"][:N])
    return gpu_engine(v, L, B, N, R, S, A, md, dtype=dtype, tanh_embed=tanh_embed)


def _assert_variant(e, variant, L):
    info = e.launch_info()
    assert info["kernel"] == {"stream": 16, "fp32_fast": 16, "lat": 18, "lat_single": 18}.get(variant, 17), info
    if variant.startswith("lat"):
        assert info["cluster"] == (3 if variant == "lat" and L >= 12 else 1), info


def _forcing(y_rows, B, N):
    """Forced history of a B-utterance launch: the oracle's trajectory on the followed rows, arbitrary codes elsewhere."""
    f = np.random.default_rng(B).integers(0, A, (B, N)).astype(np.int32)
    for i, r in enumerate(ROWS):
        if r < B:
            f[r] = y_rows[i]
    return f


@pytest.mark.parametrize("name", sorted(CONFIGS))
@pytest.mark.parametrize("variant", VARIANTS)
def test_teacher_forced_every_step(variant, name, traces, monkeypatch):
    """A launch without dumps, run_chunks(97) and the streaming call in windows of WINDOW samples, each forced with the fp32
    oracle's trajectory: every sampled index in its window of the oracle's distribution under that history."""
    L, md, N, tanh_embed, delta, max_amb = CONFIGS[name]
    w, y_or, z, _ = traces(name)
    B = _batch(variant)
    idx = [i for i, r in enumerate(ROWS) if r < B]
    rows = [ROWS[i] for i in idx]
    forced = _forcing(y_or, B, N)
    sel = w["selectors"][:N, rows]

    e = _engine(variant, w, L, B, N, md, tanh_embed, monkeypatch)
    e.set_forced(forced)
    y1 = np.zeros((B, N), np.int32)
    e.run(N, B, y1); e.synchronize()
    _assert_variant(e, variant, L)
    e.reset_history()
    y2 = np.zeros((B, N), np.int32)
    e.run_chunks(97, lambda *a: None, N, B, y2); e.synchronize()

    es = _engine(variant, w, L, B, WINDOW, md, tanh_embed, monkeypatch)
    es.reset_history()
    y3 = np.zeros((B, N), np.int32)
    ring = np.zeros((B, WINDOW), np.int32)
    for first in range(0, N, WINDOW):
        n = min(WINDOW, N - first)
        es.set_conditioning_stream(np.ascontiguousarray(w["Lh"][first:first + n, :, :B]), first)
        chunk = np.zeros((WINDOW, B), np.float32)
        chunk[:n] = w["selectors"][first:first + n, :B]
        es.set_selectors(chunk.reshape(-1))
        ring[:, :n] = forced[:, first:first + n]
        es.set_forced(ring)
        es.run_stream(first, n, B)
        es.get_yout_stream(y3[:, first:first + n], first, n)
    es.synchronize()
    _assert_variant(es, variant, L)

    for what, y in (("one launch", y1), ("run_chunks(97)", y2), (f"run_stream window {WINDOW}", y3)):
        amb = replay.check(y[rows], z[idx], sel, delta, max_amb, what=f"{variant} {name} {what}: ")
        print(f"replay {variant} {name} {what}: delta {delta} ambiguous {amb:.3f}")


def _steps(md, N):
    """Steps where the ring reads change: either side of a few dilations, maxDil and maxDil + 1, and either side of the ring's
    turns k * (maxDil + 1)."""
    s = {md, md + 1}
    for d in (2, 16, 64):
        s |= {d - 1, d, d + 1}
    for k in (1, 2, 3):
        s |= {k * (md + 1) - 1, k * (md + 1)}
    return sorted(t for t in s if t < N)


@pytest.mark.parametrize("name", sorted(CONFIGS))
@pytest.mark.parametrize("variant", VARIANTS)
def test_logits_where_ring_reads_change(variant, name, traces, monkeypatch):
    """Teacher-forced logits, dumped at the end of run_partial pieces that stop at each step of _steps, against the same trace:
    the fp16 rule against the fp32 oracle everywhere, and against the fp16-contract oracle on its prefix."""
    L, md, N, tanh_embed, delta, _ = CONFIGS[name]
    w, y_or, z, z16 = traces(name)
    B = _batch(variant)
    idx = [i for i, r in enumerate(ROWS) if r < B]
    rows = [ROWS[i] for i in idx]
    i16 = [i for i, r in enumerate(FP16_ROWS) if r < B]
    e = _engine(variant, w, L, B, N, md, tanh_embed, monkeypatch)
    e.set_forced(_forcing(y_or, B, N))
    e.reset_history()
    init, dev = 0, 0.0
    for t in _steps(md, N):
        e._samples_per_chunk = t + 1 - init
        e.run_partial(init, N, B, None, dump_activations=True)
        e._samples_per_chunk = 0
        init = t + 1
        za = e.get_za()
        _logit_check(z[idx, t], za[rows])
        dev = max(dev, replay.cdf_deviation(z[idx, t], za[rows]))
        if t < FP16_PREFIX and variant != "fp32_fast":
            _logit_check(z16[i16, t], za[[FP16_ROWS[i] for i in i16]], mean_rel=3e-4)
    _assert_variant(e, variant, L)
    print(f"logits {variant} {name}: largest CDF deviation {dev:.2e} (delta {delta})")
    assert dev <= delta / 2, f"CDF deviation {dev} leaves too little of delta {delta}"


EXPORT_ROWS_LAT = [0, 7, 8, 15, 16, 19]
EXPORT_ROWS_TC = [0, 31, 32, 63, 64, 129]
FREE_N = 800


@pytest.fixture(scope="module")
def replays():
    """Oracle traces of free-running trajectories, keyed by the rows and the trajectory itself (equal trajectories share one)."""
    cache = {}

    def get(w, rows, y, tanh_embed=False):
        L, md = CONFIGS["export"][:2]
        key = (tuple(rows), y.tobytes())
        if key not in cache:
            cache[key] = replay.oracle_trace(w, rows, (R, S, A, L, md), y.shape[1], forced=y, tanh_embed=tanh_embed)[1]
        return cache[key]
    return get


@pytest.mark.parametrize("family", ["lat", "lat_single", "tc", "stream"])
def test_free_running_replayed(family, traces, replays, monkeypatch):
    """Each kernel family generates FREE_N samples in the export configuration without forcing; its own trajectory, replayed
    through the oracle, has every sampled index in its window."""
    L, md, _, tanh_embed, delta, max_amb = CONFIGS["export"]
    w = traces("export")[0]
    B = _batch(family)
    rows = EXPORT_ROWS_TC if family == "tc" else EXPORT_ROWS_LAT
    e = _engine(family, w, L, B, FREE_N, md, tanh_embed, monkeypatch)
    y = np.zeros((B, FREE_N), np.int32)
    e.run(FREE_N, B, y); e.synchronize()
    _assert_variant(e, family, L)
    y = np.ascontiguousarray(y[rows])
    assert len(np.unique(y)) > 32
    amb = replay.check(y, replays(w, rows, y), w["selectors"][:FREE_N, rows], delta, max_amb, what=f"{family}: ")
    print(f"free-running {family}: delta {delta} ambiguous {amb:.3f}")


def _export_net(w, L, md):
    """NVWaveNet as export_weights() builds it: conv-style weights, L - 1 residual layers, no embedding tanh."""
    import torch
    from nv_wavenet_b200.nv_wavenet import NVWaveNet
    tt = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to("cuda")
    cm = lambda flat, M, K: np.ascontiguousarray(flat.reshape(K, M).T)
    dilate = [tt(np.stack([cm(w["Wprev"][l], 2 * R, R), cm(w["Wcur"][l], 2 * R, R)], axis=2)) for l in range(L)]
    return NVWaveNet(embedding_prev=tt(w["embPrev"]), embedding_curr=tt(w["embCur"]),
                     conv_out_weight=tt(cm(w["Wzs"], A, S)[:, :, None]), conv_end_weight=tt(cm(w["Wza"], A, A)[:, :, None]),
                     dilate_weights=dilate, dilate_biases=[tt(w["Bh"][l]) for l in range(L)], max_dilation=md,
                     res_weights=[tt(cm(w["Wres"][l], R, R)[:, :, None]) for l in range(L - 1)],
                     res_biases=[tt(w["Bres"][l]) for l in range(L - 1)],
                     skip_weights=[tt(cm(w["Wskip"][l], S, R)[:, :, None]) for l in range(L)],
                     skip_biases=[tt(w["Bskip"][l]) for l in range(L)], use_embed_tanh=False)


def test_nvwavenet_infer_replayed(traces, replays, monkeypatch):
    """The user path, NVWaveNet(**export-shaped weights).infer(cond, fp16=True, seed=...), without and with a window and with
    a prompt: every generated index in its window of the oracle's distribution under the Philox selectors infer() draws."""
    import torch
    for k in ("NVWN_FP16_KERNEL", "NVWN_TC_TILE", "NVWN_TC_NODUP", "NVWN_TC_FUSED", "NVWN_LAT_CLUSTER"):
        monkeypatch.delenv(k, raising=False)
    L, md, _, _, delta, max_amb = CONFIGS["export"]
    w0 = traces("export")[0]
    B, N, seed, P = B_LAT, FREE_N, 0x5EED, 150
    w = replay.sub_rows(w0, range(B))
    w["Lh"] = np.ascontiguousarray(w["Lh"][:N])
    w["selectors"] = philox_selectors(N * B, seed).reshape(N, B)
    rows = EXPORT_ROWS_LAT
    net = _export_net(w, L, md)
    cond = torch.from_numpy(np.ascontiguousarray(w["Lh"].transpose(3, 2, 1, 0))).cuda()
    y_whole = net.infer(cond, 0, seed=seed, fp16=True).cpu().numpy()
    y_win = net.infer(cond, 0, seed=seed, fp16=True, window=WINDOW).cpu().numpy()
    prompt = torch.from_numpy(np.ascontiguousarray(y_whole[:, :P]))
    y_pr = net.infer(cond, 0, seed=seed, fp16=True, prompt=prompt).cpu().numpy()
    assert np.array_equal(y_pr[:, :P], y_whole[:, :P])
    for what, y, start in (("infer", y_whole, 0), (f"infer window={WINDOW}", y_win, 0), (f"infer prompt P={P}", y_pr, P)):
        y = np.ascontiguousarray(y[rows])
        assert len(np.unique(y[:, start:])) > 32
        amb = replay.check(y, replays(w, rows, y), w["selectors"][:, rows], delta, max_amb, start=start, what=f"{what}: ")
        print(f"NVWaveNet {what}: delta {delta} ambiguous {amb:.3f}")
