"""Slot states (nvwn_save_slots / nvwn_load_slots): a slot saved at a window boundary and loaded later into another slot, or into
another engine of a different batch and window, goes on with the bits it would have had without the pause, on every engine kind; the
saved layer inputs are the history ring's, with zeros before the utterance's start; refused loads change nothing."""
import numpy as np
import pytest

from tests import refgen
from tests.test_gpu_zz_stream import A, ENV_KEYS, KINDS, L, MD, R, S

pytestmark = pytest.mark.gpu

W = 16                                   # window of the first engine; the second has W2 and another batch
W2 = 24
M = MD + 1


def _make(kind, B, N, monkeypatch, L_=L, md=MD, R_=R, S_=S, dtype=None):
    import nv_wavenet_b200 as nw
    dt, env, _, _ = KINDS[kind]
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    dtype = dtype if dtype is not None else {"fp16": nw.FP16, "fp32": nw.FP32, "fp32_fast": nw.FP32_FAST}[dt]
    return nw.NVWavenetInfer(L_, md, B, N, R=R_, S=S_, A=A, dtype=dtype)


def _lh(seed, n):
    """an utterance's conditioning [n][L][2R]"""
    return refgen.lively_inputs(seed, R, S, A, L, 1, n)["Lh"][:, :, 0]


class _Run:
    """an engine whose slots run utterances (conditioning [n][L][2R], by utterance time) window by window"""

    def __init__(self, eng, w):
        self.e, self.t = eng, 0
        eng.load(w)
        eng.reset_history()
        self.slot = {}                                                  # slot -> (lh, origin)

    def start(self, slot, lh, seed):
        self.e.restart_slots([slot], [seed])
        self.slot[slot] = (lh, self.t)

    def load(self, slot, lh, states, position):
        self.e.load_slots([slot], states)
        self.slot[slot] = (lh, self.t - position)

    def run(self, n):
        import torch
        e, t = self.e, self.t
        lh = np.zeros((n, L, e.B, 2 * R), np.float32)
        for b, (u, o) in self.slot.items():
            a = t - o
            m = max(0, min(n, len(u) - a))
            lh[:m, :, b] = u[a:a + m]
        e.set_conditioning_slots(lh, list(range(e.B)), t)
        e.set_selectors_random_slots(t, n)
        e.run_stream(t, n, e.B)
        y = torch.empty((e.B, n), dtype=torch.int32, device="cuda")
        e.get_yout_stream(y, t, n)
        self.t += n
        return y.cpu().numpy()


def _alone(kind, w, lh, seed, monkeypatch):
    """the samples an engine of this kind gives the utterance alone, from sample 0, in slot 0"""
    B = KINDS[kind][2]
    r = _Run(_make(kind, B, W, monkeypatch), w)
    r.start(0, lh, seed)
    out = np.concatenate([r.run(W)[0] for _ in range(0, len(lh), W)])[:len(lh)]
    r.e.close()
    return out


@pytest.mark.parametrize("kind", list(KINDS))
def test_round_trip_and_migration(kind, monkeypatch):
    """Slot 1's utterance is saved at t = 48, its slot runs another utterance for two windows, and it is loaded into slot 0 at
    t = 80 and continued: equal to the utterance alone.  The same state loads into a second engine of another batch and window,
    once at t0 = 24 >= maxDil and once at t0 = 5 < maxDil < 48 (every launch then reads the history at every step, and a slot that
    starts at 0 next to it still gets its own bits)."""
    w = refgen.lively_inputs(67, R, S, A, L, 1, 1)
    B = KINDS[kind][2]
    B2 = 128 if kind == "tc" else B + 3
    u, seed = _lh(1, 96), 0xA11CE
    want = _alone(kind, w, u, seed, monkeypatch)
    others = [(_lh(10 + b, 96), 500 + b) for b in range(B)]

    r = _Run(_make(kind, B, W, monkeypatch), w)
    for b in range(B):
        r.start(b, *(others[b] if b != 1 else (u, seed)))
    got = [r.run(W)[1] for _ in range(3)]
    states = r.e.save_slots([1])
    assert states.dtype.__str__() == "torch.uint8" and tuple(states.shape) == (1, r.e.slot_state_bytes())
    host = r.e.save_slots([1], out=np.empty((1, r.e.slot_state_bytes()), np.uint8))
    assert np.array_equal(host, states.cpu().numpy())
    hdr = host[0, :64]
    assert int(hdr[:4].view(np.uint32)[0]) == 0x3153564E and int(hdr[32:40].view(np.int64)[0]) == 48
    r.start(1, _lh(30, 40), 7)                                          # the slot serves another utterance meanwhile
    r.run(W); r.run(W)
    r.load(0, u, states, 48)
    got += [r.run(W)[0] for _ in range(3)]
    assert np.array_equal(np.concatenate(got), want)

    for t0 in (24, 5):
        r2 = _Run(_make(kind, B2, W2, monkeypatch), w)
        nb = _lh(40, 80)
        for b in range(B2):
            r2.start(b, *(others[b % B] if b != 2 else (nb, 99)))
        pre = r2.run(t0)
        r2.load(3, u, states, 48)
        rest = [r2.run(min(W2, 48 - k)) for k in range(0, 48, W2)]
        assert np.array_equal(np.concatenate([y[3] for y in rest]), want[48:]), t0
        neighbour = np.concatenate([pre[2]] + [y[2] for y in rest])
        assert np.array_equal(neighbour, _alone(kind, w, nb, 99, monkeypatch)[:t0 + 48]), t0
        r2.e.close()
    r.e.close()


@pytest.mark.parametrize("kind", list(KINDS))
def test_saved_inputs_are_the_ring_and_zero_before_the_start(kind, monkeypatch):
    """Each layer's saved x_l entries equal nvwn_debug_get_history at those times; a slot of a reused engine that started at sample
    0 (nvwn_reset_history leaves the ring as it was) saves zeros for its negative times."""
    import ctypes as C

    import torch
    from nv_wavenet_b200 import _lib
    lib = _lib.lib()
    w = refgen.lively_inputs(71, R, S, A, L, 1, 1)
    B = KINDS[kind][2]
    e = _make(kind, B, W, monkeypatch)
    e.load(w)
    fp16 = KINDS[kind][0] == "fp16"
    for t_end in (40, 5):                                            # the second pass reuses the ring of the first
        e.reset_history()
        lh = refgen.lively_inputs(80 + t_end, R, S, A, L, B, t_end)["Lh"]
        for first in range(0, t_end, W):
            n = min(W, t_end - first)
            e.set_conditioning_stream(lh[first:first + n], first)
            e.set_selectors_random_stream(3, first, n)
            e.run_stream(first, n, B)
        slots = [0, B - 1]
        st = e.save_slots(slots).cpu().numpy()
        hist = np.full((M, L, B, R), np.nan, np.float32)
        assert lib.nvwn_debug_get_history(e._h, C.c_void_p(hist.ctypes.data), B) == 0
        off = 64
        for l in range(L):
            d = [1, 2, 4, 8][l % 4]
            n_el = d * R
            for j, b in enumerate(slots):
                raw = st[j, off:off + n_el * (2 if fp16 else 4)]
                x = (raw.view(np.float16).astype(np.float32) if fp16 else raw.view(np.float32)).reshape(d, R)
                for k in range(d):
                    t = t_end - d + k
                    ref = hist[t % M, l, b] if t >= 0 else np.zeros(R, np.float32)
                    assert np.array_equal(x[k], ref), (t_end, l, b, t)
            off += n_el * (2 if fp16 else 4)
        assert off == st.shape[1]
        if t_end == 5:
            assert np.abs(hist[(5 - 8) % M]).max() > 0, "the ring held stale values at a negative time"
    torch.cuda.synchronize()
    e.close()


def test_refused_loads_change_nothing(monkeypatch):
    """A state of another dtype, R, L or maxDil, a bad slot list, a corrupted header: each load is refused and the run goes on with
    the bits it has without the refused calls."""
    import nv_wavenet_b200 as nw
    w = refgen.lively_inputs(67, R, S, A, L, 1, 1)
    B = KINDS["fp32"][2]
    u = _lh(1, 64)
    want = _alone("fp32", w, u, 5, monkeypatch)
    r = _Run(_make("fp32", B, W, monkeypatch), w)
    r.start(0, u, 5)
    got = [r.run(W)[0], r.run(W)[0]]
    good = r.e.save_slots([0]).cpu().numpy()
    foreign = []
    for kw in (dict(dtype=nw.FP16), dict(R_=32, S_=128), dict(L_=L + 1), dict(md=MD * 2)):
        o = _make("fp32" if "dtype" not in kw else "stream_fp16", 2, W, monkeypatch, **kw)
        o.reset_history()
        o.restart_slots([0])
        foreign.append(o.save_slots([0]).cpu().numpy())
        o.close()
    bad = good.copy()
    bad[0, :4] = 0                                                      # not a slot state
    import torch
    shifted = torch.zeros(good.size + 16, dtype=torch.uint8, device="cuda")
    misaligned = shifted[1:1 + good.size].view(1, -1)                   # device states off their 16-byte alignment
    misaligned.copy_(torch.from_numpy(good))
    with pytest.raises(nw.NvwnError, match="device states must be 16-byte aligned"):
        r.e.save_slots([0], out=misaligned)
    for states, slots, match in [(foreign[0], [1], "has dtype 1"), (foreign[1], [1], "R 32"), (foreign[2], [1], "L 13"),
                                 (foreign[3], [1], "max_dilation 16"), (bad, [1], "is not a slot state"), (good, [B], "outside"),
                                 (np.concatenate([good, good]), [1, 1], "given twice"),
                                 (misaligned, [1], "device states must be 16-byte aligned")]:
        if states.shape[1] != good.shape[1]:
            states = np.resize(states, (len(slots), good.shape[1]))             # same size, so the header check decides
        with pytest.raises(nw.NvwnError, match=match):
            r.e.load_slots(slots, states)
    with pytest.raises(ValueError, match="need 1 states"):
        r.e.load_slots([1], good[:, :-16])
    got += [r.run(W)[0] for _ in range(2)]
    assert np.array_equal(np.concatenate(got), want)
    r.e.close()
