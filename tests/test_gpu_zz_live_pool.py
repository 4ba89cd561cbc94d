"""Live serving (NVWaveNet.open_live_pool / LivePool): streams whose frames arrive at their own pace share one engine's slots, are
parked when their frames are late and resumed in any free slot, and each gets infer() of its finished frames, bit for bit, on every
engine kind; the per-slot live producer refuses what would read or overwrite a frame it no longer holds, and changes nothing then."""
import numpy as np
import pytest

from tests import refgen
from tests.common import bits_equal
from tests.test_gpu_zz_cond_slots import CC, K, STRIDE, _host, _network
from tests.test_gpu_zz_live import _refused
from tests.test_gpu_zz_selectors import _net
from tests.test_gpu_zz_slots import _store
from tests.test_gpu_zz_stream import A, ENV_KEYS, KINDS, L, MD, R, S, _engine

pytestmark = pytest.mark.gpu

W = 16
TOTALS = [30, 12, 25, 6, 40, 9, 22]                   # frames per stream; streams 3 and 5 finish early
SEEDS = [0x5000 + i for i in range(7)]


def _serve(pool, frames, rng):
    """7 streams through the pool: pushes of 0 to 3 frames per step, stream 2 stalls for five steps, stream 6 opens at step 4.
    Returns each stream's concatenated samples."""
    import torch
    ids, got, given = {}, {}, [0] * 7
    for step in range(400):
        for j in range(7):
            if j == 6 and step < 4:
                continue
            if j not in ids:
                ids[j] = pool.open(SEEDS[j])
            if j == 2 and 3 <= step < 8:
                continue
            n = min(int(rng.integers(0, 4)), TOTALS[j] - given[j])
            if n:
                piece = frames[j][:, given[j]:given[j] + n]
                pool.push(ids[j], torch.from_numpy(piece).cuda() if step % 2 else piece)
                given[j] += n
            elif given[j] == TOTALS[j] and ids[j] in pool._streams and not pool._streams[ids[j]].finished:
                pool.finish(ids[j])
        for i, y in pool.step().items():
            got.setdefault(i, []).append(y.cpu().numpy())
        if len(ids) == 7 and not pool._streams:
            break
    assert not pool._streams
    return [np.concatenate(got[ids[j]]) for j in range(7)]


@pytest.mark.parametrize("kind", list(KINDS))
def test_pool_streams_equal_infer(kind, monkeypatch):
    import torch
    import nv_wavenet_b200 as nw
    from nv_wavenet_b200.infer import live_ring_frames
    from nv_wavenet_b200.nv_wavenet import Impl, LivePool, LiveSession, NVWaveNet
    rng = np.random.default_rng(91)
    net = _network(rng)
    frames = [rng.standard_normal((CC, T)).astype(np.float32) for T in TOTALS]
    w = refgen.lively_inputs(67, R, S, A, L, 1, 1)
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    for k, v in KINDS[kind][1].items():
        monkeypatch.setenv(k, v)
    fp16 = KINDS[kind][0] == "fp16"
    slots = KINDS[kind][2]                                              # 5, or the tensor-core kernel's whole batch of 64
    if kind == "fp32_fast":
        eng = _engine(kind, W, monkeypatch)
        eng.load(w)
        eng.cond_producer_set_weights(*net, STRIDE)
        pool = LivePool(eng, CC, K, STRIDE)
    else:
        wnet = _net(w, L, R, S, A, MD)
        pool = wnet.open_live_pool(*[torch.from_numpy(a) for a in net], STRIDE, slots, W, fp16=fp16)
    got = _serve(pool, frames, np.random.default_rng(5))
    assert pool.parks > 0 and pool.resumes > 0 and pool.launches > 0
    pool.close()
    for j in range(7):
        assert got[j].shape == (TOTALS[j] * STRIDE,)
        if kind == "fp32_fast":
            one = nw.NVWavenetInfer(L, MD, 1, W, R=R, S=S, A=A, dtype=nw.FP32_FAST)
            one.load(w)
            ref = nw.NVWavenetInfer(L, MD, 1, W, R=R, S=S, A=A, dtype=nw.FP32_FAST)
            ref.load(w)
            want = torch.empty((1, TOTALS[j] * STRIDE), dtype=torch.int32, device="cuda")
            NVWaveNet._generate(ref, torch.from_numpy(_host(frames[j], net)[:, :, None]), None, SEEDS[j], None, want)
            want = want.cpu().numpy()[0]
            one.cond_producer_open_live(*net, STRIDE, live_ring_frames(W, K, STRIDE))
            live = LiveSession(one, CC, K, STRIDE, SEEDS[j], W)
        else:
            cond = torch.from_numpy(np.ascontiguousarray(_host(frames[j], net)[:, :, None].transpose(3, 2, 1, 0))).cuda()
            want = wnet.infer(cond, Impl.AUTO, seed=SEEDS[j], fp16=fp16).cpu().numpy()[0]
            live = wnet.open_live(*net, STRIDE, 1, SEEDS[j], window=W, fp16=fp16)
        y = np.concatenate([live.push(frames[j][None, :, a:a + 7]).cpu().numpy()[0] for a in range(0, TOTALS[j], 7)])
        live.close()
        assert np.array_equal(got[j], want), (kind, j, np.argwhere(got[j] != want)[:5])
        assert np.array_equal(y, want), (kind, j)
    assert len(np.unique(np.concatenate(got))) > 8


def test_pool_audio_option(monkeypatch):
    """step(audio=...) gives each stream the decoded audio of its samples."""
    import ctypes as C
    from nv_wavenet_b200 import _lib
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    rng = np.random.default_rng(93)
    net = _network(rng)
    wnet = _net(refgen.lively_inputs(73, R, S, A, L, 1, 1), L, R, S, A, MD)
    lut = np.empty(A, np.float32)
    assert _lib.lib().nvwn_mulaw_table(A, C.c_void_p(lut.ctypes.data), None, None) == 0
    pool = wnet.open_live_pool(*net, STRIDE, 3, W, fp16=True)
    i = pool.open(1)
    pool.push(i, rng.standard_normal((CC, 5)).astype(np.float32))
    y, audio = pool.step(audio="float")
    assert set(y) == set(audio) == {i} and np.array_equal(audio[i], lut[y[i].cpu().numpy()])
    pool.close()


def test_live_slot_refusals_change_nothing(monkeypatch):
    """A push past a slot's ring, a production that reads frames that have left it, a push to a slot with no live utterance and
    nvwn_cond_producer_set_slots in live mode are refused; the store is as it was, and the productions that follow give the
    conditioning of the frames on the host, bit for bit."""
    from nv_wavenet_b200.infer import live_ring_frames
    B, N = KINDS["fp32"][2], 24
    rng = np.random.default_rng(97)
    net = _network(rng)
    frames = rng.standard_normal((CC, 12)).astype(np.float32)
    e = _engine("fp32", N, monkeypatch)
    e.set_conditioning(np.zeros((N, L, B, 2 * R), np.float32), 0, N)
    e.cond_producer_set_weights(*net, STRIDE)
    ring = live_ring_frames(N, K, STRIDE)
    assert ring == 8
    _refused(e.cond_producer_attach_live, [1], [0], [0], [frames[:, :2]], match="not in live mode")
    e.cond_producer_open_live_slots(ring)
    _refused(e.cond_producer_set_slots, [0], [frames], [0], match="live mode")
    _refused(e.cond_producer_push_slots, [1], [frames[:, :1]], match="slot 1 has no live utterance")
    e.cond_producer_attach_live([1], [0], [0], [frames[:, :ring]])
    _refused(e.cond_producer_push_slots, [1], [frames[:, ring:ring + 1]], match="1 frames would overwrite frame 0 of slot 1")
    e.cond_producer_run_slots([1], 0, 20)
    e.synchronize()
    before = _store(e)
    e.cond_producer_push_slots([1], [frames[:, ring:ring + 2]])          # samples from 20 read frames 2 ..
    _refused(e.cond_producer_push_slots, [1], [frames[:, ring + 2:ring + 3]], match="would overwrite frame 2")
    _refused(e.cond_producer_run_slots, [1], 0, 5, match="frame 0, which sample 0 of slot 1's utterance reads, has left the ring")
    e.synchronize()
    assert bits_equal(_store(e), before)
    e.cond_producer_run_slots([1], 20, 24)
    e.synchronize()
    got, host = _store(e), _host(frames[:, :ring + 2], net)
    for t in range(20, 44):
        want = host[t] if t < (ring + 2) * STRIDE else np.zeros((L, 2 * R), np.float32)
        assert bits_equal(got[t % N, :, 1], want), t
    # a resumed utterance: sample 0 before the engine's, frames from 3 on
    e.cond_producer_attach_live([2], [-20], [3], [frames[:, 3:9]])
    _refused(e.cond_producer_run_slots, [2], 0, 4, match="frame 2, which sample 20 of slot 2's utterance reads")
    e.cond_producer_run_slots([2], 5, 10)                                # samples 25 .. 34 read frames 3 ..
    e.synchronize()
    got, host = _store(e), _host(frames[:, :9], net)
    for t in range(5, 15):
        assert bits_equal(got[t % N, :, 2], host[t + 20]), t
