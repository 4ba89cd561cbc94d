"""Streaming generation (nvwn_run_stream): an engine of W samples whose buffers are rings generates any length bit-identically to
one engine that holds the whole length -- samples and last-step dumps -- on every kernel."""
import numpy as np
import pytest

from tests import refgen
from tests.common import bits_equal

pytestmark = pytest.mark.gpu

R, S, A = 64, 256, 256
L, MD = 12, 8                       # L = 12: the cluster kernel's shortest stack; history ring of MD + 1 = 9 slots
T = 40
SEED = 0x5EED0123
# kind -> (dtype name, environment at creation, batch, expected launch info)
KINDS = {
    "lat_cluster": ("fp16", {"NVWN_FP16_KERNEL": "lat"}, 5, {"kernel": 18, "cluster": 3}),
    "lat_single": ("fp16", {"NVWN_FP16_KERNEL": "lat", "NVWN_LAT_CLUSTER": "0"}, 5, {"kernel": 18, "cluster": 1}),
    "tc": ("fp16", {"NVWN_FP16_KERNEL": "tc"}, 64, {"kernel": 17}),
    "stream_fp16": ("fp16", {"NVWN_FP16_KERNEL": "stream"}, 5, {"kernel": 16}),
    "fp32": ("fp32", {}, 5, {"kernel": 16}),
    "fp32_fast": ("fp32_fast", {}, 5, {"kernel": 16}),
}
ENV_KEYS = ("NVWN_FP16_KERNEL", "NVWN_LAT_CLUSTER", "NVWN_TC_TILE", "NVWN_TC_NODUP", "NVWN_TC_FUSED", "NVWN_LAT_MAX_B")


def _engine(kind, n, monkeypatch, L_=L, md=MD):
    import nv_wavenet_b200 as nw
    dt, env, B, _ = KINDS[kind]
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    dtype = {"fp16": nw.FP16, "fp32": nw.FP32, "fp32_fast": nw.FP32_FAST}[dt]
    return nw.NVWavenetInfer(L_, md, B, n, R=R, S=S, A=A, dtype=dtype)


def _ranges(total, W):
    """Uneven ranges of at most W samples: some of exactly W, some crossing the wrap."""
    sizes = [W, max(1, W - 2), 1, W, (W + 1) // 2, 2]
    out, first, i = [], 0, 0
    while first < total:
        n = min(sizes[i % len(sizes)], total - first)
        out.append((first, n))
        first += n; i += 1
    return out


def _full(kind, w, B, monkeypatch, forced=None):
    e = _engine(kind, T, monkeypatch)
    e.load(w)
    e.set_inputs(w["Lh"], w["selectors"])
    e.set_selectors_random(SEED)
    if forced is not None:
        e.set_forced(forced)
    y = np.zeros((B, T), np.int32)
    e.run(T, B, y, dump_activations=True); e.synchronize()
    return y, e.activations(), e


def _windowed(kind, w, B, W, monkeypatch, forced=None):
    e = _engine(kind, W, monkeypatch)
    e.load(w)
    e.reset_history()
    y = np.zeros((B, T), np.int32)
    ring = np.zeros((B, W), np.int32)
    ranges = _ranges(T, W)
    for first, n in ranges:
        e.set_conditioning_stream(w["Lh"][first:first + n], first)
        e.set_selectors_random_stream(SEED, first, n)
        if forced is not None:
            for t in range(first, first + n):
                ring[:, t % W] = forced[:, t]
            e.set_forced(ring)
        e.run_stream(first, n, B, dump_activations=(first + n == T))
        e.get_yout_stream(y[:, first:first + n], first, n)
    e.synchronize()
    return y, e.activations(), e, ranges


def _assert_same(a, b):
    ya, da = a[0], a[1]
    yb, db = b[0], b[1]
    assert np.array_equal(ya, yb), np.argwhere(ya != yb)[:5]
    for k in ("xt", "skip", "zs", "za", "p"):
        assert bits_equal(da[k], db[k]), k


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_window_invariance(kind, monkeypatch):
    B, want = KINDS[kind][2], KINDS[kind][3]
    w = refgen.lively_inputs(21, R, S, A, L, B, T)
    full = _full(kind, w, B, monkeypatch)
    assert len(np.unique(full[0])) > 8
    info = full[2].launch_info()
    assert all(info[k] == v for k, v in want.items()), info
    for W in (3, 7, 13, T):                     # 3; shorter than the history ring (9); longer, not dividing T; the whole length
        got = _windowed(kind, w, B, W, monkeypatch)
        if W < T:
            assert any(n == W for _, n in got[3]) and any(f % W + n > W for f, n in got[3])
        assert all(got[2].launch_info()[k] == v for k, v in want.items())
        _assert_same(full, got)


@pytest.mark.parametrize("kind", ["lat_cluster", "stream_fp16", "fp32"])
def test_teacher_forcing_through_a_window(kind, monkeypatch):
    B = KINDS[kind][2]
    w = refgen.lively_inputs(22, R, S, A, L, B, T)
    forced = np.random.default_rng(3).integers(0, A, (B, T)).astype(np.int32)
    _assert_same(_full(kind, w, B, monkeypatch, forced), _windowed(kind, w, B, 7, monkeypatch, forced))


@pytest.mark.parametrize("kind", ["lat_cluster", "lat_single", "tc", "fp32"])
def test_classic_run_then_stream_continues(kind, monkeypatch):
    B = KINDS[kind][2]
    N = 17
    w = refgen.lively_inputs(23, R, S, A, L, B, 2 * N)
    e2 = _engine(kind, 2 * N, monkeypatch)
    e2.load(w); e2.set_inputs(w["Lh"], w["selectors"]); e2.set_selectors_random(SEED)
    want = np.zeros((B, 2 * N), np.int32)
    e2.run(2 * N, B, want, dump_activations=True); e2.synchronize()

    e = _engine(kind, N, monkeypatch)
    e.load(w); e.set_inputs(w["Lh"][:N], w["selectors"][:N]); e.set_selectors_random(SEED)
    got = np.zeros((B, 2 * N), np.int32)
    e.run(N, B)
    e.get_yout_stream(got[:, :N], 0, N)
    e.set_conditioning_stream(w["Lh"][N:], N)
    e.set_selectors_random_stream(SEED, N, N)
    e.run_stream(N, N, B, dump_activations=True)
    e.get_yout_stream(got[:, N:], N, N); e.synchronize()
    _assert_same((want, e2.activations()), (got, e.activations()))


def test_errors(monkeypatch):
    import nv_wavenet_b200 as nw
    B, N = 5, 8
    w = refgen.lively_inputs(24, R, S, A, L, B, N)
    e = _engine("fp32", N, monkeypatch)
    e.load(w); e.set_inputs(w["Lh"], w["selectors"])

    def bad(fn, *args, match):
        with pytest.raises(nw.NvwnError, match=match) as ex:
            fn(*args)
        assert "(code -1)" in str(ex.value)

    bad(e.run_stream, 3, 2, B, match="next sample is 0")
    e.run_stream(0, 5, B)
    bad(e.run_stream, 4, 2, B, match="next sample is 5")
    bad(e.run_stream, 6, 2, B, match="next sample is 5")
    e.run_stream(5, 8, B)
    bad(e.run_stream, 5, 1, B, match="next sample is 13")
    e.reset_history()
    e.run_stream(0, 1, B)
    e.run(N, B)                                  # a classic run moves the next sample to its end
    e.run_stream(N, 1, B)
    bad(e.run_stream, N + 1, N + 1, B, match="count <= num_samples")
    bad(e.run_stream, N + 1, -1, B, match="count <= num_samples")
    bad(e.run_stream, -1, 1, B, match="first_sample >= 0")
    bad(e.run_stream, N + 1, 1, 0, match="batch_size")
    bad(e.run_stream, N + 1, 1, B + 1, match="batch_size")
    e.run_stream(N + 1, 1, B - 1)                # fewer utterances than the engine holds: allowed off the tensor-core path
    bad(e.set_selectors_random_stream, 1, 0, N + 1, match="num_samples")
    bad(e.set_selectors_random_stream, 1, -1, 1, match="first_sample")

    t = _engine("tc", 4, monkeypatch)
    wt = refgen.lively_inputs(25, R, S, A, L, 64, 4)
    t.load(wt); t.set_inputs(wt["Lh"], wt["selectors"])
    bad(t.run_stream, 0, 2, 63, match="tensor-core path needs batch_size")
    t.run_stream(0, 2, 64)


def test_c3_long_form_with_the_producer_on_a_side_stream(monkeypatch):
    """C3 model (L20, maxDil 512, B = 64), 3 x 16 000 + 123 samples through a window of 4 096, conditioning produced per window on
    a side stream: equal to one engine of the whole length filled by set_conditioning_from_features."""
    import torch
    import nv_wavenet_b200 as nw
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    L3, md, B, W = 20, 512, 64, 4096
    Cc, stride, window = 80, 9, 27
    frames = 5347
    total = frames * stride
    assert total == 3 * 16000 + 123
    w = refgen.lively_inputs(26, R, S, A, L3, 1, 1)
    rng = np.random.default_rng(27)
    feats = rng.standard_normal((B, Cc, frames), dtype=np.float32)
    wu = (0.1 * rng.standard_normal((Cc, Cc, window))).astype(np.float32)
    bu = (0.1 * rng.standard_normal(Cc)).astype(np.float32)
    wc = (0.2 * rng.standard_normal((L3 * 2 * R, Cc))).astype(np.float32)
    bc = (0.05 * rng.standard_normal(L3 * 2 * R)).astype(np.float32)
    args = (feats, wu, bu, wc, bc, stride)

    full = nw.NVWavenetInfer(L3, md, B, total, R=R, S=S, A=A, dtype=nw.FP16)
    full.load(w); full.reset_history()
    full.set_conditioning_from_features(*args)
    full.set_selectors_random(SEED)
    want = torch.empty((B, total), dtype=torch.int32, device="cuda")
    full.run(total, B, want); torch.cuda.synchronize()
    want = want.cpu().numpy()
    del full

    e = nw.NVWavenetInfer(L3, md, B, W, R=R, S=S, A=A, dtype=nw.FP16)
    e.load(w); e.reset_history()
    assert e.cond_producer_load(*args) == total
    side, gen = torch.cuda.Stream(), torch.cuda.Stream()
    got = torch.empty((B, total), dtype=torch.int32, device="cuda")
    done = []
    for k, first in enumerate(range(0, total, W // 2)):     # two chunks per window: one is produced while the other is generated
        n = min(W // 2, total - first)
        if k >= 2:
            side.wait_event(done[k - 2])         # the chunk whose positions it overwrites has been generated and read
        e.cond_producer_run_stream(first, n, stream=side)
        ready = torch.cuda.Event(); ready.record(side)
        gen.wait_event(ready)
        e.set_selectors_random_stream(SEED, first, n, stream=gen)
        e.run_stream(first, n, B, stream=gen)
        e.get_yout_stream(got[:, first:first + n], first, n, stream=gen)
        done.append(torch.cuda.Event()); done[-1].record(gen)
    torch.cuda.synchronize()
    assert e.launch_info()["cluster"] == 3
    got = got.cpu().numpy()
    assert len(np.unique(want)) > 16
    assert np.array_equal(got, want), np.argwhere(got != want)[:5]


@pytest.mark.parametrize("fp16", [False, True])
def test_nvwavenet_infer_window(fp16):
    import ctypes as C
    import torch
    from nv_wavenet_b200.nv_wavenet import Impl
    from tests.test_gpu_zz_selectors import _net
    Lm, B, md = 4, 3, 4
    w = refgen.lively_inputs(28, R, S, A, Lm, B, 1300)
    net = _net(w, Lm, R, S, A, md)
    cond = torch.from_numpy(np.ascontiguousarray(w["Lh"].transpose(3, 2, 1, 0))).cuda()
    for seed in (None, 9):
        for n in (1300, 700):
            c = cond[..., :n].contiguous()
            libc = C.CDLL(None)
            libc.srand(77); want = net.infer(c, Impl.AUTO, seed=seed, fp16=fp16).cpu().numpy()
            libc.srand(77); got = net.infer(c, Impl.AUTO, seed=seed, fp16=fp16, window=512).cpu().numpy()
            assert np.array_equal(want, got) and len(np.unique(want)) > 8
    net = _net(w, Lm, R, S, A, md)
    net.infer(cond[..., :900].contiguous(), Impl.AUTO, seed=1, fp16=fp16, window=512)
    net.infer(cond[..., :1100].contiguous(), Impl.AUTO, seed=1, fp16=fp16, window=512)
    assert net.engines_created == 1                   # one engine of 512 samples serves every length
