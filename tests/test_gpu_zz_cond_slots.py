"""Per-slot conditioning producer (nvwn_cond_producer_set_weights / _set_slots / _run_slots) and NVWaveNet.infer_many_from_features:
each slot's conditioning made on the device from its own utterance's mel frames must equal the host restatement of that utterance
alone (nvwn_cond_from_features_host), bit for bit in fp32, and the fp16 stores what the per-slot upload of those rows leaves."""
import ctypes as C

import numpy as np
import pytest

from tests import refgen
from tests.common import bits_equal
from tests.test_gpu_zz_selectors import _net
from tests.test_gpu_zz_slots import L, MD, _batch, _eng, _slots_of, _store
from tests.test_gpu_zz_stream import A, ENV_KEYS, R, S

pytestmark = pytest.mark.gpu

CC, K, STRIDE = 6, 12, 5                 # upsampling window 12: not a multiple of the stride


def _network(rng, Lm=L, Cc=CC, k=K):
    """upsample_weight [C][C][window], upsample_bias [C], cond_weight [L*2R][C], cond_bias [L*2R]: conditioning of order 1"""
    return ((rng.standard_normal((Cc, Cc, k)) / np.sqrt(Cc * k / STRIDE)).astype(np.float32),
            (0.1 * rng.standard_normal(Cc)).astype(np.float32),
            (0.5 * rng.standard_normal((Lm * 2 * R, Cc)) / np.sqrt(Cc)).astype(np.float32),
            (0.1 * rng.standard_normal(Lm * 2 * R)).astype(np.float32))


def _host(frames, net, stride=STRIDE, Lm=L):
    """nvwn_cond_from_features_host of one utterance alone: [T * stride][L][2R]"""
    from nv_wavenet_b200 import _lib
    wu, bu, wc, bc = net
    Cc, T = frames.shape
    out = np.full((T * stride, Lm, 1, 2 * R), np.nan, np.float32)
    p = lambda a: C.c_void_p(np.ascontiguousarray(a, np.float32).ctypes.data)
    f = np.ascontiguousarray(frames, np.float32)
    assert _lib.lib().nvwn_cond_from_features_host(p(out), C.c_void_p(f.ctypes.data), 1, Cc, T, p(wu), p(bu), wu.shape[2], stride, p(wc), p(bc),
                                                    Lm, R) == 0
    return out[:, :, 0]


def _utterances(rng, counts, Cc=CC):
    return [rng.standard_normal((Cc, T)).astype(np.float32) for T in counts]


@pytest.mark.parametrize("kind", ["fp32", "lat_cluster", "tc", "stream_fp16"])
def test_per_slot_production_equals_host_rows(kind, monkeypatch):
    """Three utterances of different lengths and starts in slot 0, a row in 8-15 of a 16-row tile and the last slot; the range
    produced in uneven pieces, one across the ring wrap; a utterance ending inside the range.  fp32: the store equals the host rows
    (0 past each end) bit for bit, every other row keeps its contents.  Every kind: the store equals what
    nvwn_set_conditioning_slots leaves for those fp32 rows (compared through the fp32 readback, which is exact for fp16)."""
    import torch
    B, N = _batch(kind), 24
    rng = np.random.default_rng(7)
    net = _network(rng)
    slots = _slots_of(kind)
    frames = _utterances(rng, [7, 3, 9])
    starts = [0, 9, 4]                                              # the second ends at 24, inside the produced range
    host = [_host(f, net) for f in frames]
    base = rng.standard_normal((N, L, B, 2 * R)).astype(np.float32)
    pieces = [(13, 5), (18, 10), (28, 1), (29, 8)]                  # absolute samples [13, 37); (18, 10) crosses the wrap at 24
    want = base.copy()
    rows = np.zeros((37, L, len(slots), 2 * R), np.float32)
    for i, (s, t0, h) in enumerate(zip(slots, starts, host)):
        for t in range(13, 37):
            rows[t, :, i] = h[t - t0] if t - t0 < len(h) else 0.0
            want[t % N, :, s] = rows[t, :, i]

    e = _eng(kind, B, N, monkeypatch)
    e.set_conditioning(base, 0, N)
    e.cond_producer_set_weights(*net, STRIDE)
    keep = e.cond_producer_set_slots(slots[::-1], [torch.from_numpy(f).cuda() for f in frames[::-1]], starts[::-1])   # device frames
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    for first, n in pieces:
        e.cond_producer_run_slots(slots, first, n, stream=side)
    side.synchronize()
    del keep
    got = _store(e)
    assert np.isfinite(got).all()
    if kind == "fp32":
        assert bits_equal(got, want), np.argwhere(got.view(np.uint32) != want.view(np.uint32))[:5]

    e2 = _eng(kind, B, N, monkeypatch)
    e2.set_conditioning(base, 0, N)
    for first, n in pieces:
        e2.set_conditioning_slots(np.ascontiguousarray(rows[first:first + n]), slots, first)
    torch.cuda.synchronize()
    ref = _store(e2)
    assert bits_equal(got, ref), np.argwhere(got.view(np.uint32) != ref.view(np.uint32))[:5]


def _plan_has_restarts(lengths, slots, window):
    from nv_wavenet_b200.nv_wavenet import plan_slots
    starts = {t for _, t in plan_slots(lengths, slots, window)}
    return len(starts - {0}) >= 3


@pytest.mark.parametrize("fp16", [False, True])
def test_infer_many_from_features_equals_infer(fp16, monkeypatch):
    import torch
    from nv_wavenet_b200.nv_wavenet import Impl
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    rng = np.random.default_rng(17)
    counts = [1, 3, 20, 13, 41, 7, 30]                              # 5 .. 205 samples; windows of 64
    lengths = [T * STRIDE for T in counts]
    assert _plan_has_restarts(lengths, 3, 64) and any(n % 64 for n in lengths)
    seeds = [301 + 13 * u for u in range(len(counts))]
    w = refgen.lively_inputs(19, R, S, A, L, 1, 1)
    wnet = _net(w, L, R, S, A, MD)
    cnet = _network(rng)
    frames = _utterances(rng, counts)
    # host frames for some utterances, CUDA ones for the others; torch weights
    feats = [torch.from_numpy(f).cuda() if u % 2 else f for u, f in enumerate(frames)]
    timing = {}
    got = wnet.infer_many_from_features(feats, seeds, *[torch.from_numpy(a) for a in cnet], STRIDE, slots=3, window=64, fp16=fp16,
                                        timing=timing)
    assert set(timing) == {"produce_s", "produce_wait_s", "restart_select_s", "generate_s"} and timing["produce_s"] > 0
    conds = [torch.from_numpy(np.ascontiguousarray(_host(f, cnet).transpose(2, 1, 0))).cuda() for f in frames]      # [2R][L][n]
    many = wnet.infer_many(conds, seeds, slots=3, window=64, fp16=fp16)
    for u, c in enumerate(conds):
        want = wnet.infer(c[:, None].contiguous(), Impl.AUTO, seed=seeds[u], fp16=fp16)[0].cpu().numpy()
        assert got[u].shape == (lengths[u],)
        assert np.array_equal(got[u].cpu().numpy(), want), (u, np.argwhere(got[u].cpu().numpy() != want)[:5])
        assert np.array_equal(many[u].cpu().numpy(), want), u
    assert len(np.unique(got[4].cpu().numpy())) > 8


def test_infer_many_from_features_c3(monkeypatch):
    """C3 model (L20, maxDil 512), 64 slots, 80 channels, upsampling window 800, stride 200; 72 utterances of 5-40 frames through
    windows of 2 048.  Six of them equal infer_many on conditioning expanded by the whole-batch producer on one-utterance engines."""
    import torch
    import nv_wavenet_b200 as nw
    from nv_wavenet_b200 import _lib
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    L3, md, Cc, k, stride, W = 20, 512, 80, 800, 200, 2048
    rng = np.random.default_rng(23)
    counts = [int(v) for v in rng.integers(5, 41, 72)]
    seeds = [int(v) for v in rng.integers(0, 2 ** 62, 72)]
    wu = (rng.standard_normal((Cc, Cc, k)) / np.sqrt(Cc * k / stride)).astype(np.float32)
    bu = (0.1 * rng.standard_normal(Cc)).astype(np.float32)
    wc = (0.5 * rng.standard_normal((L3 * 2 * R, Cc)) / np.sqrt(Cc)).astype(np.float32)
    bc = (0.1 * rng.standard_normal(L3 * 2 * R)).astype(np.float32)
    frames = [torch.from_numpy(f).cuda() for f in _utterances(rng, counts, Cc)]
    w = refgen.lively_inputs(29, R, S, A, L3, 1, 1)
    wnet = _net(w, L3, R, S, A, md)
    got = wnet.infer_many_from_features(frames, seeds, wu, bu, wc, bc, stride, slots=64, window=W, fp16=True)
    assert wnet._engine(64, 2 * W, True).launch_info()["cluster"] == 3
    lib = _lib.lib()
    lib.nvwn_debug_get_conditioning.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    subset = sorted(int(u) for u in rng.choice(72, 6, replace=False))
    conds = []
    for u in subset:
        n = counts[u] * stride
        one = nw.NVWavenetInfer(L3, md, 1, n, R=R, S=S, A=A, dtype=nw.FP32)
        assert one.set_conditioning_from_features(frames[u][None].contiguous(), wu, bu, wc, bc, stride) == n
        lh = np.full((n, L3, 1, 2 * R), np.nan, np.float32)
        assert lib.nvwn_debug_get_conditioning(one._h, C.c_void_p(lh.ctypes.data), 0, n) == 0
        conds.append(torch.from_numpy(np.ascontiguousarray(lh[:, :, 0].transpose(2, 1, 0))).cuda())
        one.close()
    want = wnet.infer_many(conds, [seeds[u] for u in subset], slots=64, window=W, fp16=True)
    for i, u in enumerate(subset):
        assert len(np.unique(want[i].cpu().numpy())) > 16
        assert np.array_equal(got[u].cpu().numpy(), want[i].cpu().numpy()), (u, np.argwhere(got[u].cpu().numpy() != want[i].cpu().numpy())[:5])


def _serve_engine(kind, side_stream, monkeypatch):
    """Four windows of W = 16 through an engine of 2W, slots restarted at window boundaries; the conditioning producer one window
    ahead on a side stream ordered only by events, or on the generating stream just before each window."""
    import torch
    B, W = _batch(kind), 16
    rng = np.random.default_rng(37)
    net = _network(rng)
    w = refgen.lively_inputs(41, R, S, A, L, B, 1)
    e = _eng(kind, B, 2 * W, monkeypatch)
    e.load(w)
    e.reset_history()
    e.cond_producer_set_weights(*net, STRIDE)
    first_frames = _utterances(rng, [int(v) for v in rng.integers(2, 14, B)])
    later = {2 * W: ([1, B - 1], _utterances(rng, [9, 4])), 3 * W: ([0], _utterances(rng, [3]))}
    attach = {0: (list(range(B)), first_frames), **later}
    cur = torch.cuda.current_stream()
    side = torch.cuda.Stream() if side_stream else cur
    side.wait_stream(cur)
    ready, read = {}, {}

    def produce(k):
        if k - 2 in read:
            side.wait_event(read[k - 2])
        if k * W in attach:
            sl, fr = attach[k * W]
            e.cond_producer_set_slots(sl, fr, [k * W] * len(sl), stream=side)
        e.cond_producer_run_slots(range(B), k * W, W, stream=side)
        ready[k] = torch.cuda.Event()
        ready[k].record(side)

    y = np.zeros((B, 4 * W), np.int32)
    if side_stream:
        produce(0)
    for k in range(4):
        if side_stream:
            cur.wait_event(ready[k])
        else:
            produce(k)
        if k * W in attach:
            sl = attach[k * W][0]
            e.restart_slots(sl, [1000 + 7 * s + k for s in sl])
        e.set_selectors_random_slots(k * W, W)
        e.run_stream(k * W, W, B)
        read[k] = torch.cuda.Event()
        read[k].record(cur)
        if side_stream and k + 1 < 4:
            produce(k + 1)
        e.get_yout_stream(y[:, k * W:(k + 1) * W], k * W, W)
    torch.cuda.synchronize()
    return y


@pytest.mark.parametrize("kind", ["lat_cluster", "fp32"])
def test_side_stream_one_window_ahead_equals_in_order(kind, monkeypatch):
    y_side = _serve_engine(kind, True, monkeypatch)
    y_inline = _serve_engine(kind, False, monkeypatch)
    assert np.array_equal(y_side, y_inline) and len(np.unique(y_side)) > 8


def test_errors(monkeypatch):
    import nv_wavenet_b200 as nw
    from nv_wavenet_b200 import _lib
    lib = _lib.lib()
    B, N = 5, 8
    rng = np.random.default_rng(43)
    net = _network(rng)
    f = _utterances(rng, [2, 3])
    e = _eng("fp32", B, N, monkeypatch)

    def bad(fn, *args, match):
        with pytest.raises(nw.NvwnError, match=match) as ex:
            fn(*args)
        assert "(code -1)" in str(ex.value)

    bad(e.cond_producer_run_slots, [0], 0, 1, match="nvwn_cond_producer_run_slots: nvwn_cond_producer_set_weights has not been called")
    bad(e.cond_producer_set_slots, [0], f[:1], [0], match="nvwn_cond_producer_set_slots: nvwn_cond_producer_set_weights has not been called")
    wu, bu, wc, bc = net
    bad(lambda: _lib.check(lib.nvwn_cond_producer_set_weights(e._h, CC, C.c_void_p(wu.ctypes.data), C.c_void_p(bu.ctypes.data), 4, 5,
                                                              C.c_void_p(wc.ctypes.data), C.c_void_p(bc.ctypes.data), None), "w"),
        match="nvwn_cond_producer_set_weights: bad sizes")                # window < stride
    e.cond_producer_set_weights(*net, STRIDE)
    bad(e.cond_producer_run_slots, [1], 0, 1, match="nvwn_cond_producer_run_slots: slot 1 has no frames attached")
    e.cond_producer_set_slots([1, 3], f, [2, 0])
    e.cond_producer_run_slots([1, 3], 2, N)
    bad(e.cond_producer_run_slots, [1, 3], 1, 1, match="nvwn_cond_producer_run_slots: first_sample 1 is before the start 2 of slot 1")
    bad(e.cond_producer_run_slots, [3], 0, N + 1, match="nvwn_cond_producer_run_slots: need first_sample >= 0 and 0 <= num_samples")
    bad(e.cond_producer_run_slots, [3], -1, 1, match="nvwn_cond_producer_run_slots: need first_sample >= 0")
    for name, call in {"nvwn_cond_producer_run_slots": lambda sl: e.cond_producer_run_slots(sl, 2, 1),
                       "nvwn_cond_producer_set_slots": lambda sl: e.cond_producer_set_slots(sl, [f[0]] * len(sl), [2] * len(sl))}.items():
        bad(call, list(range(B + 1)), match=f"{name}: need 1 <= n <= B")
        bad(call, [0, -1], match=f"{name}: slot -1 is outside")
        bad(call, [B], match=f"{name}: slot {B} is outside")
        bad(call, [1, 3, 1], match=f"{name}: slot 1 is given twice")
    slots = (C.c_int * 1)(2)
    counts = (C.c_int * 1)(0)
    starts = (C.c_longlong * 1)(0)
    ptrs = (C.c_void_p * 1)(f[0].ctypes.data)
    bad(lambda: _lib.check(lib.nvwn_cond_producer_set_slots(e._h, slots, 1, ptrs, counts, starts, None), "s"),
        match="nvwn_cond_producer_set_slots: utterance 0 \\(slot 2\\) has num_frames = 0")
    counts[0], ptrs[0] = 2, None
    bad(lambda: _lib.check(lib.nvwn_cond_producer_set_slots(e._h, slots, 1, ptrs, counts, starts, None), "s"),
        match="nvwn_cond_producer_set_slots: the frames of utterance 0 \\(slot 2\\) are NULL")
    starts[0], ptrs[0] = -1, f[0].ctypes.data
    bad(lambda: _lib.check(lib.nvwn_cond_producer_set_slots(e._h, slots, 1, ptrs, counts, starts, None), "s"),
        match="nvwn_cond_producer_set_slots: utterance 0 \\(slot 2\\) starts at -1")
    with pytest.raises(ValueError):
        e.cond_producer_set_slots([0, 1], f[:1], [0, 0])                 # one frame array per slot
    with pytest.raises(ValueError):
        e.cond_producer_set_slots([0], [f[0][None]], [0])                # frames are [C][T]
    # a producer slot call counts as a per-slot call: a smaller batch is refused until reset_history, which forgets the frames
    bad(e.run_stream, 0, 4, 2, match="nvwn_run_stream: after a per-slot call")
    e.reset_history()
    e.run_stream(0, 4, 2)
    bad(e.cond_producer_run_slots, [3], 0, 1, match="nvwn_cond_producer_run_slots: slot 3 has no frames attached")
    e.cond_producer_set_slots([4], f[1:], [0])
    bad(e.run_stream, 4, 1, 2, match="nvwn_run_stream: after a per-slot call")
    e.reset_history()
    e.run_stream(0, 1, 2)
    e.cond_producer_set_slots([4], f[1:], [0])
    e.reset_history()
    e.cond_producer_set_weights(*net, STRIDE)
    bad(e.cond_producer_run_slots, [4], 0, 1, match="nvwn_cond_producer_run_slots: slot 4 has no frames attached")
    e.cond_producer_set_slots([4], f[1:], [0])
    e.cond_producer_set_weights(*net, STRIDE)                              # new weights forget the frames as well
    bad(e.cond_producer_run_slots, [4], 0, 1, match="nvwn_cond_producer_run_slots: slot 4 has no frames attached")
    e.cond_producer_set_slots([4], f[1:], [0])
    e.cond_producer_run_slots([4], 0, 0)                                   # an empty range is valid
    bad(e.run_stream, 0, 1, 2, match="nvwn_run_stream: after a per-slot call")
    e.synchronize()


def test_host_arrays_may_be_reused_on_return(monkeypatch):
    """Slots, frame pointers, counts, starts and the frames themselves in pinned host memory, overwritten as soon as each call
    returns, leave the store that ordinary arrays leave."""
    import torch
    from nv_wavenet_b200 import _lib
    lib = _lib.lib()
    B, N = 5, 32
    rng = np.random.default_rng(47)
    net = _network(rng)
    frames = _utterances(rng, [5, 4])
    stores = []
    for pinned in (False, True):
        e = _eng("fp32", B, N, monkeypatch)
        e.set_conditioning(np.zeros((N, L, B, 2 * R), np.float32), 0, N)
        e.cond_producer_set_weights(*net, STRIDE)
        if pinned:
            pf = [torch.from_numpy(f).pin_memory() for f in frames]
            slots = torch.tensor([3, 0], dtype=torch.int32).pin_memory()
            ptrs = torch.tensor([t.data_ptr() for t in pf], dtype=torch.int64).pin_memory()
            counts = torch.tensor([5, 4], dtype=torch.int32).pin_memory()
            starts = torch.tensor([0, 6], dtype=torch.int64).pin_memory()
            p = lambda t: C.c_void_p(t.data_ptr())
            assert lib.nvwn_cond_producer_set_slots(e._h, p(slots), 2, p(ptrs), p(counts), p(starts), None) == 0
            for t in pf:
                t.fill_(1e6)
            counts.fill_(1); starts.fill_(0)
            slots[:] = torch.tensor([0, 3], dtype=torch.int32)
            assert lib.nvwn_cond_producer_run_slots(e._h, p(slots), 2, 6, N, None) == 0
            slots.fill_(-1)
        else:
            e.cond_producer_set_slots([3, 0], frames, [0, 6])
            e.cond_producer_run_slots([0, 3], 6, N)
        torch.cuda.synchronize()
        stores.append(_store(e))
    assert bits_equal(stores[0], stores[1]) and np.abs(stores[0]).max() > 0.1
