"""The whole-batch conditioning producer (nvwn_cond_producer_load / _run) and the per-slot one (nvwn_cond_producer_set_weights /
_set_slots / _run_slots) are two instances of one producer: calls of the two sets, interleaved on one engine with networks of
different channel counts, must each leave the store their producer leaves alone, and a whole batch of utterances must give the
same store bits through either producer."""
import ctypes as C

import numpy as np
import pytest

from tests.common import bits_equal
from tests.test_gpu_zz_cond_slots import _host, _network
from tests.test_gpu_zz_slots import L, _batch, _eng, _slots_of, _store
from tests.test_gpu_zz_stream import R

pytestmark = pytest.mark.gpu

KINDS = ["fp32", "stream_fp16", "tc", "lat_cluster"]
N = 24
CC_A, K_A, STRIDE_A, T_A = 6, 12, 5, 2          # whole batch: positions [0, 10) of every row
CC_B, K_B, STRIDE_B = 4, 10, 4                  # per slot: absolute samples [12, 24) of three rows
SLOT_FRAMES, SLOT_STARTS = [4, 3, 1], [0, 8, 12]    # ends at 16, 20 and 16: inside the produced range
S_FIRST = 12


def _host_batch(features, net, stride):
    """nvwn_cond_from_features_host of a whole batch: [T * stride][L][B][2R]"""
    from nv_wavenet_b200 import _lib
    wu, bu, wc, bc = net
    B, Cc, T = features.shape
    out = np.full((T * stride, L, B, 2 * R), np.nan, np.float32)
    p = lambda a: C.c_void_p(np.ascontiguousarray(a, np.float32).ctypes.data)
    f = np.ascontiguousarray(features, np.float32)
    assert _lib.lib().nvwn_cond_from_features_host(p(out), C.c_void_p(f.ctypes.data), B, Cc, T, p(wu), p(bu), wu.shape[2], stride, p(wc), p(bc),
                                                    L, R) == 0
    return out


def _inputs(kind):
    B = _batch(kind)
    rng = np.random.default_rng(53)
    net_a, net_b = _network(rng, Cc=CC_A, k=K_A), _network(rng, Cc=CC_B, k=K_B)
    feats = [rng.standard_normal((B, CC_A, T_A)).astype(np.float32) for _ in range(2)]
    frames = [rng.standard_normal((CC_B, T)).astype(np.float32) for T in SLOT_FRAMES]
    return B, net_a, net_b, feats, frames


def _whole(s):
    return s[:T_A * STRIDE_A]


def _rows(s, slots):
    return s[S_FIRST:, :, slots]


@pytest.mark.parametrize("kind", KINDS)
def test_interleaved_producers_keep_their_own_network(kind, monkeypatch):
    B, net_a, net_b, feats, frames = _inputs(kind)
    slots = _slots_of(kind)
    n_w, n_s = T_A * STRIDE_A, N - S_FIRST
    zeros = np.zeros((N, L, B, 2 * R), np.float32)

    # what each producer leaves alone, on a fresh engine
    alone_w = []
    for f in feats:
        e = _eng(kind, B, N, monkeypatch)
        e.set_conditioning(zeros, 0, N)
        assert e.cond_producer_load(f, *net_a, STRIDE_A) == n_w
        e.cond_producer_run(0, n_w)
        e.synchronize()
        alone_w.append(_whole(_store(e)))
        e.close()
    e = _eng(kind, B, N, monkeypatch)
    e.set_conditioning(zeros, 0, N)
    e.cond_producer_set_weights(*net_b, STRIDE_B)
    e.cond_producer_set_slots(slots, frames, SLOT_STARTS)
    e.cond_producer_run_slots(slots, S_FIRST, n_s)
    e.synchronize()
    alone_s = _rows(_store(e), slots)
    e.close()
    if kind == "fp32":
        for f, a in zip(feats, alone_w):
            assert bits_equal(a, _host_batch(f, net_a, STRIDE_A))
        want = np.zeros_like(alone_s)
        for i, (fr, t0) in enumerate(zip(frames, SLOT_STARTS)):
            h = _host(fr, net_b, STRIDE_B)
            for t in range(S_FIRST, N):
                if t - t0 < len(h):
                    want[t - S_FIRST, :, i] = h[t - t0]
        assert bits_equal(alone_s, want)
    assert np.abs(alone_s).max() > 0.1 and np.abs(alone_w[0]).max() > 0.1 and not bits_equal(alone_w[0], alone_w[1])

    def check(whole=None, per_slot=True):
        e.synchronize()
        got = _store(e)
        if whole is not None:
            assert bits_equal(_whole(got), alone_w[whole])
        if per_slot:
            assert bits_equal(_rows(got, slots), alone_s)

    def wipe():
        e.set_conditioning(zeros, 0, N)

    e = _eng(kind, B, N, monkeypatch)
    wipe()
    e.cond_producer_load(feats[0], *net_a, STRIDE_A)
    e.cond_producer_set_weights(*net_b, STRIDE_B)
    e.cond_producer_set_slots(slots, frames, SLOT_STARTS)
    e.cond_producer_run_slots(slots, S_FIRST, n_s)
    check()
    e.cond_producer_run(0, n_w)
    check(whole=0)
    e.cond_producer_load(feats[1], *net_a, STRIDE_A)                   # new features: the per-slot network and frames stay
    wipe()
    e.cond_producer_run_slots(slots, S_FIRST, n_s)
    check()
    e.cond_producer_run(0, n_w)
    check(whole=1)
    e.reset_history()                                                  # forgets the per-slot utterances only
    wipe()
    e.cond_producer_run(0, n_w)
    check(whole=1, per_slot=False)
    import nv_wavenet_b200 as nw
    with pytest.raises(nw.NvwnError, match="has no frames attached"):
        e.cond_producer_run_slots(slots, S_FIRST, n_s)
    e.cond_producer_set_slots(slots, frames, SLOT_STARTS)
    e.cond_producer_run_slots(slots, S_FIRST, n_s)
    check(whole=1)


@pytest.mark.parametrize("kind", KINDS)
def test_whole_batch_equals_every_slot(kind, monkeypatch):
    """features [B][C][T] through nvwn_cond_producer_load / _run, and features[b] attached to slot b and produced for all B slots,
    leave the same store bits."""
    B, net_a, _, feats, _ = _inputs(kind)
    first, n = 3, T_A * STRIDE_A
    stores = []
    for whole in (True, False):
        e = _eng(kind, B, N, monkeypatch)
        e.set_conditioning(np.zeros((N, L, B, 2 * R), np.float32), 0, N)
        if whole:
            e.cond_producer_load(feats[0], *net_a, STRIDE_A)
            e.cond_producer_run(0, n, first_sample=first)
        else:
            e.cond_producer_set_weights(*net_a, STRIDE_A)
            e.cond_producer_set_slots(list(range(B)), list(feats[0]), [first] * B)
            e.cond_producer_run_slots(list(range(B)), first, n)
        e.synchronize()
        stores.append(_store(e))
        e.close()
    assert np.abs(stores[0]).max() > 0.1
    assert bits_equal(stores[0], stores[1])
