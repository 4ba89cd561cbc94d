"""Slot states of scored prompts (nvwn_score_save_states): the state of a scoring row equals, byte for byte, the state nvwn_save_slots
writes of a slot primed from that row (nvwn_prime_slots_from_score), on all three fp16 kernel families, with the prompt shorter and
longer than maxDil; its header fields; zeros at negative times; host and device destinations; and every refusal leaves the scoring
stream, and what it scores next, unchanged."""
import numpy as np
import pytest

from tests import refgen
from tests.test_gpu_zz_park import _make
from tests.test_gpu_zz_stream import A, L, MD, R, S

pytestmark = pytest.mark.gpu

W = 16
FP16_KINDS = ["lat_cluster", "tc", "stream_fp16"]
BS = 3                                                   # rows of the scoring stream


def _layers():
    """per layer (its body offset in bytes, d_l)"""
    out, off, d = [], 64, 1
    for _ in range(L):
        out.append((off, d))
        off += d * R * 2
        d = 1 if 2 * d > MD else 2 * d
    return out


def _score(e, codes, lh, first, n):
    """scores samples [first, first + n) of the rows: conditioning lh [P][L][Bs][2R] at positions t mod W"""
    full = np.zeros((n, L, e.B, 2 * R), np.float32)
    full[:, :, :codes.shape[0]] = lh[first:first + n]
    pos = first % W
    assert pos + n <= W
    e.set_conditioning(full, pos, n)
    return e.score_stream(codes[:, first:first + n], first)


def _score_to(e, codes, lh, P):
    for first in range(0, P, W):
        _score(e, codes, lh, first, min(W, P - first))


def _inputs(P, seed):
    rng = np.random.default_rng(seed)
    codes = rng.integers(0, A, (BS, P + W)).astype(np.int32)
    lh = refgen.lively_inputs(seed, R, S, A, L, BS, P + W)["Lh"]                       # [n][L][Bs][2R]
    return codes, lh


@pytest.mark.parametrize("kind", FP16_KINDS)
@pytest.mark.parametrize("P", [5, 37])
def test_states_equal_prime_then_save(kind, P, monkeypatch):
    """Rows 2 and 0 after a prompt of P samples (5 < maxDil = 8 < 37): device and host states are equal, and equal the states
    of slots primed from those rows; the header holds the engine's sizes, P, the rows' last two codes and the seeds; a layer's
    times before 0 are zero."""
    import nv_wavenet_b200 as nw
    w = refgen.lively_inputs(67, R, S, A, L, 1, 1)
    B = 64 if kind == "tc" else 5
    e = _make(kind, B, W, monkeypatch)
    e.load(w)
    codes, lh = _inputs(P, 100 + P)
    _score_to(e, codes, lh, P)
    rows, seeds = [2, 0], [0x1234_5678_9ABC_DEF0, 22]
    dev = e.score_save_states(rows, seeds)
    host = e.score_save_states(rows, seeds, out=np.empty((2, e.slot_state_bytes()), np.uint8))
    got = dev.cpu().numpy()
    assert np.array_equal(got, host)
    e.reset_history()
    e.prime_slots_from_score(rows, [1, 3], seeds)
    want = e.save_slots([1, 3]).cpu().numpy()
    assert np.array_equal(got, want), np.argwhere(got != want)[:8]
    no_seed = e.score_save_states(rows).cpu().numpy()
    assert not no_seed[:, 40:48].any() and np.array_equal(np.delete(no_seed, np.s_[40:48], axis=1), np.delete(got, np.s_[40:48], axis=1))
    for j, r in enumerate(rows):
        h = got[j, :64]
        i32 = h[:32].view(np.int32)
        assert int(h[:4].view(np.uint32)[0]) == 0x3153564E
        assert list(i32[1:5]) == [nw.FP16, R, L, MD]
        prev = codes[r, P - 2] if P >= 2 else 128
        assert (int(i32[5]), int(i32[6]), int(i32[7])) == (prev, codes[r, P - 1], 0)
        assert int(h[32:40].view(np.int64)[0]) == P
        assert int(h[40:48].view(np.uint64)[0]) == seeds[j] & (2 ** 64 - 1)
        assert not h[48:64].any()
        for off, d in _layers():
            body = got[j, off:off + d * R * 2].reshape(d, R * 2)
            assert not body[:max(0, d - P)].any(), (off, d)                      # times P - d .. -1
            if d <= P:
                assert body.any()
    e.close()


def _refused(code, fn, *args):
    import nv_wavenet_b200 as nw
    with pytest.raises(nw.NvwnError) as ex:
        fn(*args)
    assert f"(code {code})" in str(ex.value)


def test_refusals_change_nothing(monkeypatch):
    """Rows outside [0, Bs), a row given twice, NULL arguments, no open stream, a packed stream and an fp32 engine are refused;
    the stream goes on to score the next window with the bits of an engine that never saw them, and its states are unchanged."""
    import ctypes as C
    from nv_wavenet_b200 import _lib
    w = refgen.lively_inputs(67, R, S, A, L, 1, 1)
    P = 21
    codes, lh = _inputs(P, 7)
    clean = _make("lat_cluster", 5, W, monkeypatch)
    clean.load(w)
    _score_to(clean, codes, lh, P)
    want_states = clean.score_save_states([0, 1, 2]).cpu().numpy()
    want = _score(clean, codes, lh, P, W - P % W)

    e = _make("lat_cluster", 5, W, monkeypatch)
    e.load(w)
    _refused(-1, e.score_save_states, [0])                                        # no open stream
    _score_to(e, codes, lh, P)
    _refused(-1, e.score_save_states, [BS])
    _refused(-1, e.score_save_states, [-1])
    _refused(-1, e.score_save_states, [1, 1])
    import torch
    shifted = torch.zeros(e.slot_state_bytes() + 16, dtype=torch.uint8, device="cuda")
    _refused(-1, e.score_save_states, [0], None, shifted[1:1 + e.slot_state_bytes()].view(1, -1))     # device states off 16 bytes
    out = np.empty((1, e.slot_state_bytes()), np.uint8)
    lib = _lib.lib()
    row = np.zeros(1, np.int32)
    assert lib.nvwn_score_save_states(e._h, None, 1, None, C.c_void_p(out.ctypes.data), None) == -1
    assert lib.nvwn_score_save_states(e._h, C.c_void_p(row.ctypes.data), 1, None, None, None) == -1
    assert lib.nvwn_score_save_states(e._h, C.c_void_p(row.ctypes.data), 0, None, C.c_void_p(out.ctypes.data), None) == -1
    assert lib.nvwn_score_save_states(None, C.c_void_p(row.ctypes.data), 1, None, C.c_void_p(out.ctypes.data), None) == -1
    assert np.array_equal(e.score_save_states([0, 1, 2]).cpu().numpy(), want_states)
    got = _score(e, codes, lh, P, W - P % W)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))

    packed = _make("lat_cluster", 5, W, monkeypatch)
    packed.load(w)
    packed.set_conditioning(np.zeros((W, L, 5, 2 * R), np.float32), 0, W)
    packed.score_stream_packed(codes[:, :W], np.zeros((BS, W), np.uint8), 0)
    _refused(-2, packed.score_save_states, [0])
    f32 = _make("lat_cluster", 5, W, monkeypatch, dtype=_lib.FP32)
    f32.load(w)
    _refused(-2, f32.score_save_states, [0])
    for x in (clean, e, packed, f32):
        x.close()
