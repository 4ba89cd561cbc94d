"""Continuous batching: restarting single slots of a running streaming engine (nvwn_restart_slots), per-slot conditioning and
selectors, and NVWaveNet.infer_many on top of them.  A restarted slot must continue exactly as a fresh engine started with its
utterance, and the slots that were not restarted exactly as if nothing had happened, on every kernel."""
import ctypes as C

import numpy as np
import pytest

from tests import refgen
from tests.common import bits_equal
from tests.test_gpu_zz_selectors import _net, philox_selectors
from tests.test_gpu_zz_stream import A, ENV_KEYS, KINDS, R, S, _engine

pytestmark = pytest.mark.gpu

L, MD, T = 12, 8, 60                    # history ring of MD + 1 = 9 slots


def _batch(kind):
    """Utterances of the test engines: two 16-row tiles for the latency and plain kernels (so rows 8-15 of a tile take part), one
    64-utterance tile for the tensor-core kernel, which takes whole batches only."""
    return 64 if kind == "tc" else 20


def _slots_of(kind):
    """slot 0, a row in 8-15 of a 16-row tile, the last slot"""
    return [0, 37, 63] if kind == "tc" else [0, 11, 19]


def _eng(kind, B, n, monkeypatch):
    import nv_wavenet_b200 as nw
    if B == KINDS[kind][2]:
        return _engine(kind, n, monkeypatch)
    dt, env, _, _ = KINDS[kind]
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    dtype = {"fp16": nw.FP16, "fp32": nw.FP32, "fp32_fast": nw.FP32_FAST}[dt]
    return nw.NVWavenetInfer(L, MD, B, n, R=R, S=S, A=A, dtype=dtype)


def _ranges(W, breaks):
    """launch ranges of at most W samples that also end at every restart time in `breaks`"""
    out, first = [], 0
    while first < T:
        nxt = min([first + W, T] + [t for t in breaks if t > first])
        out.append((first, nxt - first))
        first = nxt
    return out


def _rows(a, keep, axis):
    return np.take(a, keep, axis=axis)


def _run_slots(kind, w, W, base_seeds, restarts, monkeypatch):
    """Generates T samples in ranges of at most W, restarting slots at the times of `restarts` ({t0: [(slot, seed, cond)]}).
    Conditioning goes in through set_conditioning_slots in two groups of slots, selectors through set_selectors_random_slots."""
    B = _batch(kind)
    e = _eng(kind, B, W, monkeypatch)
    e.load(w)
    e.reset_history()
    e.restart_slots(range(B), base_seeds)                 # every slot starts its utterance at 0 with its own seed
    lh = w["Lh"].copy()                                    # [T][L][B][2R]: what each slot is conditioned on, restarts merged
    group = [_slots_of(kind)[2], _slots_of(kind)[0], _slots_of(kind)[1]]
    rest = [b for b in range(B) if b not in group]
    y = np.zeros((B, T), np.int32)
    for first, n in _ranges(W, sorted(restarts)):
        if first in restarts:
            starts = restarts[first]
            e.restart_slots([s for s, _, _ in starts], [seed for _, seed, _ in starts])
            for s, _, c in starts:
                lh[first:, :, s] = c[:T - first]
        for g in (group, rest):
            e.set_conditioning_slots(np.ascontiguousarray(lh[first:first + n][:, :, g]), g, first)
        e.set_selectors_random_slots(first, n)
        e.run_stream(first, n, B, dump_activations=(first + n == T))
        e.get_yout_stream(y[:, first:first + n], first, n)
    e.synchronize()
    return y, e.activations()


def _fresh(kind, w, slot, seed, cond, count, monkeypatch):
    """A fresh engine of the same kind and batch, started at 0 with utterance `cond` in `slot` under `seed`: count samples."""
    B = _batch(kind)
    e = _eng(kind, B, T, monkeypatch)
    e.load(w)
    lh = w["Lh"].copy()
    lh[:len(cond), :, slot] = cond
    sel = np.repeat(philox_selectors(T, 0)[:, None], B, axis=1)
    sel[:, slot] = philox_selectors(T, seed)
    e.set_inputs(lh, np.ascontiguousarray(sel))
    y = np.zeros((B, count), np.int32)
    e.run(count, B, y)
    e.synchronize()
    return y[slot]


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_restart_equals_a_fresh_start(kind, monkeypatch):
    B = _batch(kind)
    s0, s1, s2 = _slots_of(kind)
    w = refgen.lively_inputs(31, R, S, A, L, B, T)
    rng = np.random.default_rng(32)
    cond = lambda: (0.5 * rng.standard_normal((T, L, 2 * R))).astype(np.float32)
    base_seeds = [0x1000 + 7 * b for b in range(B)]
    # restarts before maxDil, in the middle, and the same slot (s1) a second time
    restarts = {3: [(s0, 0xDEADBEEF12345678, cond()), (s1, 77, cond())], 20: [(s2, 2 ** 40 + 5, cond())], 33: [(s1, 91, cond())]}
    utterances = []                                        # (slot, t0, seed, cond, length)
    for t0 in sorted(restarts):
        for s, seed, c in restarts[t0]:
            later = [t for t in restarts if t > t0 and any(x[0] == s for x in restarts[t])]
            utterances.append((s, t0, seed, c, (min(later) if later else T) - t0))
    fresh = {(s, t0): _fresh(kind, w, s, seed, c, n, monkeypatch) for s, t0, seed, c, n in utterances}
    keep = [b for b in range(B) if b not in (s0, s1, s2)]
    for W in (7, 16):                                      # 7: shorter than the history ring
        y, act = _run_slots(kind, w, W, base_seeds, restarts, monkeypatch)
        y0, act0 = _run_slots(kind, w, W, base_seeds, {}, monkeypatch)
        assert len(np.unique(y)) > 8
        for s, t0, seed, c, n in utterances:
            got = y[s, t0:t0 + n]
            assert np.array_equal(got, fresh[(s, t0)]), (W, s, t0, np.argwhere(got != fresh[(s, t0)])[:5])
        assert np.array_equal(y[keep], y0[keep]), np.argwhere(y[keep] != y0[keep])[:5]
        for k, axis in (("xt", 1), ("skip", 1), ("zs", 0), ("za", 0), ("p", 0)):
            assert bits_equal(_rows(act[k], keep, axis), _rows(act0[k], keep, axis)), (W, k)


def _store(e):
    from nv_wavenet_b200 import _lib
    lib = _lib.lib()
    lib.nvwn_debug_get_conditioning.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    got = np.full((e.N, e.L, e.B, 2 * e.R), np.nan, np.float32)
    assert lib.nvwn_debug_get_conditioning(e._h, C.c_void_p(got.ctypes.data), 0, e.N) == 0
    return got


@pytest.mark.parametrize("kind", ["lat_single", "tc", "stream_fp16", "fp32"])
def test_conditioning_slots_write_only_their_rows(kind, monkeypatch):
    import torch
    B, N = _batch(kind), 16
    rng = np.random.default_rng(41)
    base = rng.standard_normal((N, L, B, 2 * R)).astype(np.float32)
    e = _eng(kind, B, N, monkeypatch)
    e.set_conditioning(base, 0, N)
    merged = base.copy()
    writes = [([B - 1, 0, 9], 3 * N + 11, 9, False),      # positions 11..15 and 0..3: across the wrap, host source
              ([5, 2], 5 * N + 15, 2, True),              # positions 15 and 0, device source
              (list(range(B)), 7, 4, False)]              # every slot
    for slots, first, n, on_device in writes:
        new = rng.standard_normal((n, L, len(slots), 2 * R)).astype(np.float32)
        e.set_conditioning_slots(torch.from_numpy(new).cuda() if on_device else new, slots, first)
        for i in range(n):
            merged[(first + i) % N][:, slots] = new[i]
    torch.cuda.synchronize()
    e2 = _eng(kind, B, N, monkeypatch)
    e2.set_conditioning(merged, 0, N)
    got, want = _store(e), _store(e2)
    assert np.isfinite(got).all()
    assert bits_equal(got, want), np.argwhere(got.view(np.uint32) != want.view(np.uint32))[:5]


def test_conditioning_slots_fp32_host_source_over_several_staging_chunks(monkeypatch):
    """On an fp32 engine a host source reaches the row conversion through the 64 MB staging buffer: a source of more samples than
    one chunk holds, across the wrap, leaves the same store as the same values from device memory, and the values themselves."""
    import torch
    B, N, shift = 8, 1500, 100
    slots = [7, 0, 3, 5, 1, 6, 2, 4]
    new = np.random.default_rng(43).standard_normal((N, L, B, 2 * R)).astype(np.float32)
    assert new[:N - shift].nbytes > 64 << 20                              # the piece before the wrap takes two chunks
    want = np.empty_like(new)
    want[:, :, slots] = new
    want = np.roll(want, shift, axis=0)                                   # sample N + shift + i sits at position (shift + i) mod N
    for src in (new, torch.from_numpy(new).cuda()):
        e = _eng("fp32", B, N, monkeypatch)
        e.set_conditioning_slots(src, slots, N + shift)
        torch.cuda.synchronize()
        assert bits_equal(_store(e), want), "host" if src is new else "device"
        e.close()


def test_selectors_per_slot(monkeypatch):
    """Per-slot selectors equal the host restatement (counter t - origin, key seed) and a one-utterance engine's stream draw."""
    B, W, Tn = 5, 16, 40
    w = refgen.lively_inputs(51, R, S, A, L, B, Tn)
    seeds0 = [11, 12, 13, 14, 15]
    restarts = {10: ([1, 4], [2 ** 63 + 3, 99]), 13: ([2], [123456789])}
    breaks = sorted(restarts)

    def run(host_selectors):
        e = _eng("fp32", B, W, monkeypatch)
        e.load(w)
        e.reset_history()
        e.restart_slots(range(B), seeds0)
        origin, seed = [0] * B, list(seeds0)
        y = np.zeros((B, Tn), np.int32)
        first = 0
        while first < Tn:
            n = min([first + W, Tn] + [t for t in breaks if t > first]) - first
            if first in restarts:
                sl, sd = restarts[first]
                e.restart_slots(sl, sd)
                for s, k in zip(sl, sd):
                    origin[s], seed[s] = first, k
            e.set_conditioning_stream(w["Lh"][first:first + n], first)
            if host_selectors:
                sel = np.zeros((W, B), np.float32)
                for b in range(B):
                    draw = philox_selectors(first + n - origin[b], seed[b])[first - origin[b]:]
                    for i in range(n):
                        sel[(first + i) % W, b] = draw[i]
                e.set_selectors(sel)
            else:
                e.set_selectors_random_slots(first, n)
            e.run_stream(first, n, B)
            e.get_yout_stream(y[:, first:first + n], first, n)
            first += n
        e.synchronize()
        return y

    y = run(False)
    assert np.array_equal(y, run(True)) and len(np.unique(y)) > 8
    # slot 4 from t0 = 10 against a one-utterance engine drawing set_selectors_random_stream(99, t - 10)
    one = _eng("fp32", 1, W, monkeypatch)
    one.load(w)
    one.reset_history()
    y1 = np.zeros((1, Tn - 10), np.int32)
    for first in range(0, Tn - 10, W):
        n = min(W, Tn - 10 - first)
        one.set_conditioning_stream(np.ascontiguousarray(w["Lh"][10 + first:10 + first + n, :, 4:5]), first)
        one.set_selectors_random_stream(99, first, n)
        one.run_stream(first, n, 1)
        one.get_yout_stream(y1[:, first:first + n], first, n)
    one.synchronize()
    assert np.array_equal(y1[0], y[4, 10:])


def _utterances(seed, lengths, Lm):
    import torch
    w = refgen.lively_inputs(seed, R, S, A, Lm, len(lengths), max(lengths))
    conds = [torch.from_numpy(np.ascontiguousarray(w["Lh"][:n, :, u].transpose(2, 1, 0))).cuda() for u, n in enumerate(lengths)]
    return w, conds


@pytest.mark.parametrize("fp16", [False, True])
def test_infer_many_equals_infer(fp16, monkeypatch):
    from nv_wavenet_b200.nv_wavenet import Impl
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    lengths = [1, 5, 37, 513, 700, 1300, 2049]
    seeds = [101 + 17 * u for u in range(len(lengths))]
    w, conds = _utterances(61, lengths, L)
    net = _net(w, L, R, S, A, MD)
    got = net.infer_many(conds, seeds, slots=3, window=512, fp16=fp16)
    created = net.engines_created
    again = net.infer_many(conds[::-1], seeds[::-1], slots=3, window=512, fp16=fp16)
    assert net.engines_created == created                 # the second call reuses the engine
    for u, c in enumerate(conds):
        want = net.infer(c[:, None].contiguous(), Impl.AUTO, seed=seeds[u], fp16=fp16)[0].cpu().numpy()
        assert np.array_equal(got[u].cpu().numpy(), want), (u, np.argwhere(got[u].cpu().numpy() != want)[:5])
        assert np.array_equal(again[len(conds) - 1 - u].cpu().numpy(), want), u
    assert len(np.unique(got[-1].cpu().numpy())) > 8


def test_infer_many_c3(monkeypatch):
    """C3 model (L20, maxDil 512) with 64 slots and a window of 4 096: 80 utterances of 2 000 - 20 000 samples; six of them, chosen
    by seed, are bit-identical to infer() alone."""
    import torch
    from nv_wavenet_b200.nv_wavenet import Impl
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    L3, md = 20, 512
    rng = np.random.default_rng(71)
    lengths = [int(v) for v in rng.integers(2000, 20001, 80)]
    offsets = [int(v) for v in rng.integers(0, 20000, 80)]
    seeds = [int(v) for v in rng.integers(0, 2 ** 62, 80)]
    w = refgen.lively_inputs(72, R, S, A, L3, 1, 1)
    g = torch.Generator(device="cuda").manual_seed(73)
    base = 0.5 * torch.randn((2 * R, L3, 40000), generator=g, device="cuda")
    conds = [base[:, :, o:o + n] for o, n in zip(offsets, lengths)]
    net = _net(w, L3, R, S, A, md)
    got = net.infer_many(conds, seeds, slots=64, window=4096, fp16=True)
    assert net._engine(64, 4096, True).launch_info()["cluster"] == 3
    for u in sorted(rng.choice(80, 6, replace=False)):
        want = net.infer(conds[u][:, None].contiguous(), Impl.AUTO, seed=seeds[u], fp16=True)[0].cpu().numpy()
        assert len(np.unique(want)) > 16
        assert np.array_equal(got[u].cpu().numpy(), want), (u, np.argwhere(got[u].cpu().numpy() != want)[:5])


def test_errors(monkeypatch):
    import nv_wavenet_b200 as nw
    from nv_wavenet_b200 import _lib
    lib = _lib.lib()
    B, N = 5, 8
    e = _eng("fp32", B, N, monkeypatch)
    lh = np.zeros((2, L, 1, 2 * R), np.float32)

    def bad(fn, *args, match):
        with pytest.raises(nw.NvwnError, match=match) as ex:
            fn(*args)
        assert "(code -1)" in str(ex.value)

    def bad_c(rc, match):
        assert rc == -1
        assert match in lib.nvwn_last_error().decode()

    one = (C.c_int * 1)(0)
    bad_c(lib.nvwn_restart_slots(None, one, 1, None, None), "nvwn_restart_slots: NULL engine")
    bad_c(lib.nvwn_restart_slots(e._h, None, 1, None, None), "nvwn_restart_slots: slots is NULL")
    bad_c(lib.nvwn_set_conditioning_slots(None, C.c_void_p(lh.ctypes.data), one, 1, 0, 1, None), "nvwn_set_conditioning_slots: NULL engine")
    bad_c(lib.nvwn_set_conditioning_slots(e._h, None, one, 1, 0, 1, None), "nvwn_set_conditioning_slots: Lh is NULL")
    bad_c(lib.nvwn_set_conditioning_slots(e._h, C.c_void_p(lh.ctypes.data), None, 1, 0, 1, None), "nvwn_set_conditioning_slots: slots is NULL")
    bad_c(lib.nvwn_set_conditioning_slots(e._h, C.c_void_p(lh.ctypes.data), one, 1, 0, -1, None), "nvwn_set_conditioning_slots: need")
    bad_c(lib.nvwn_set_selectors_random_slots(None, 0, 1, None), "nvwn_set_selectors_random_slots: NULL engine")
    bad_c(lib.nvwn_set_conditioning_slots(e._h, C.c_void_p(lh.ctypes.data), one, 0, 0, 1, None), "nvwn_set_conditioning_slots: need 1 <= n <= B")
    bad(e.restart_slots, [], match="nvwn_restart_slots: need 1 <= n <= B")
    calls = {"nvwn_restart_slots": lambda slots: e.restart_slots(slots),
             "nvwn_set_conditioning_slots": lambda slots: e.set_conditioning_slots(
                 np.zeros((2, L, len(slots), 2 * R), np.float32), slots, 0)}
    for name, call in calls.items():
        bad(call, list(range(B + 1)), match=f"{name}: need 1 <= n <= B")
        bad(call, [0, -1], match=f"{name}: slot -1 is outside")
        bad(call, [B], match=f"{name}: slot {B} is outside")
        bad(call, [1, 3, 1], match=f"{name}: slot 1 is given twice")
    with pytest.raises(ValueError):
        e.restart_slots([0, 1], [5])                      # one seed per slot
    bad(e.set_conditioning_slots, lh, [0], -1, match="nvwn_set_conditioning_slots: need first_sample >= 0")
    bad(e.set_conditioning_slots, np.zeros((N + 1, L, 1, 2 * R), np.float32), [0], 0, match="nvwn_set_conditioning_slots: need")
    bad(e.set_selectors_random_slots, -1, 1, match="nvwn_set_selectors_random_slots: need first_sample >= 0")
    bad(e.set_selectors_random_slots, 0, N + 1, match="nvwn_set_selectors_random_slots: need")
    bad(e.set_selectors_random_slots, 0, -1, match="nvwn_set_selectors_random_slots: need")
    # Lh must be [n][L][len(slots)][2R]: a mismatch is refused before anything reads past the array
    for shape in ((2, L, 2, 2 * R), (2, L + 1, 1, 2 * R), (2, L, 1, R), (2, L, 2 * R)):
        with pytest.raises(ValueError, match="set_conditioning_slots: Lh must be"):
            e.set_conditioning_slots(np.zeros(shape, np.float32), [0], 0)
    # what is valid: an empty range, a whole ring
    e.restart_slots([B - 1, 0], [1, 2])
    e.set_conditioning_slots(np.zeros((N, L, 2, 2 * R), np.float32), [3, 4], 5)
    e.set_selectors_random_slots(3, N)
    e.set_selectors_random_slots(3, 0)
    # the rows of the per-slot calls are laid out for runs of the whole batch: a smaller batch is refused until reset_history
    bad(e.run_stream, 0, 4, 2, match="nvwn_run_stream: after a per-slot call .* runs need batch_size equal to the engine's batch size")
    bad(e.run_partial, 0, 4, 2, match="nvwn_run_partial: after a per-slot call")
    e.run_stream(0, 4, B)
    e.set_inputs(np.zeros((N, L, B, 2 * R), np.float32), np.full((N, B), 0.5, np.float32))     # resets the history
    e.run_stream(0, 4, 2)
    e.restart_slots([4])
    bad(e.run_stream, 4, 1, 2, match="nvwn_run_stream: after a per-slot call")
    e.set_selectors_random_slots(4, 1)
    e.run_stream(4, 1, B)
    e.reset_history()
    e.set_selectors_random_slots(0, 1)
    bad(e.run_stream, 0, 1, 3, match="nvwn_run_stream: after a per-slot call")
    e.synchronize()


def test_slot_arrays_are_copied_before_return(monkeypatch):
    """Slots and seeds in pinned host memory, overwritten right after nvwn_restart_slots returns, give the samples of the same
    restart from ordinary arrays."""
    import torch
    from nv_wavenet_b200 import _lib
    lib = _lib.lib()
    B, N = 5, 16
    w = refgen.lively_inputs(81, R, S, A, L, B, N)
    ys = []
    for pinned in (False, True):
        e = _eng("fp32", B, N, monkeypatch)
        e.load(w)
        e.set_conditioning(w["Lh"], 0, N)
        e.reset_history()
        e.restart_slots(range(B), [3, 4, 5, 6, 7])
        e.set_selectors_random_slots(0, 6)
        e.run_stream(0, 6, B)
        if pinned:
            slots = torch.tensor([3, 1], dtype=torch.int32).pin_memory()
            seeds = torch.tensor([2 ** 40 + 9, 77], dtype=torch.int64).pin_memory()
            assert lib.nvwn_restart_slots(e._h, C.c_void_p(slots.data_ptr()), 2, C.c_void_p(seeds.data_ptr()), None) == 0
            slots.fill_(0); seeds.fill_(0)                 # the caller reuses its arrays at once
        else:
            e.restart_slots([3, 1], [2 ** 40 + 9, 77])
        e.set_selectors_random_slots(6, N - 6)
        e.run_stream(6, N - 6, B)
        y = np.zeros((B, N), np.int32)
        e.get_yout(y, 0, N)
        e.synchronize()
        ys.append(y)
    assert np.array_equal(ys[0], ys[1]) and len(np.unique(ys[0])) > 8
