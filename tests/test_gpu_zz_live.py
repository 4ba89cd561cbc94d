"""Live vocoding (nvwn_cond_producer_open_live / _push, NVWaveNet.open_live): mel frames pushed a few at a time into a ring on the
device give, push by push, the samples infer() gives the finished utterance, bit for bit, on every engine kind; the ring producer
leaves the store a loaded producer leaves; refused calls change nothing."""
import ctypes as C

import numpy as np
import pytest

from tests import refgen
from tests.common import bits_equal
from tests.test_gpu_zz_cond_slots import CC, K, STRIDE, _network
from tests.test_gpu_zz_selectors import _net
from tests.test_gpu_zz_slots import _store
from tests.test_gpu_zz_stream import A, ENV_KEYS, KINDS, L, MD, R, S, _engine

pytestmark = pytest.mark.gpu

W = 24                                   # generation window; the upsampling window K = 12 is not a multiple of STRIDE = 5
SEED = 0x11FE


def _host_batch(frames, net):
    """nvwn_cond_from_features_host of frames [B][C][T]: [T * stride][L][B][2R]"""
    from nv_wavenet_b200 import _lib
    wu, bu, wc, bc = net
    B, Cc, T = frames.shape
    out = np.full((T * STRIDE, L, B, 2 * R), np.nan, np.float32)
    p = lambda a: C.c_void_p(np.ascontiguousarray(a, np.float32).ctypes.data)
    f = np.ascontiguousarray(frames, np.float32)
    assert _lib.lib().nvwn_cond_from_features_host(p(out), C.c_void_p(f.ctypes.data), B, Cc, T, p(wu), p(bu), K, STRIDE, p(wc), p(bc), L, R) == 0
    return out


def _refused(fn, *args, match):
    import nv_wavenet_b200 as nw
    with pytest.raises(nw.NvwnError, match=match) as ex:
        fn(*args)
    assert "(code -1)" in str(ex.value)


@pytest.mark.parametrize("kind", list(KINDS))
def test_live_pushes_equal_infer(kind, monkeypatch):
    """Pushes of 0, 1, 1, 4, 3, 15 (more than the ring of 8 frames), 2 and 14 frames: generation pieces cross the window's wrap at
    multiples of 24.  The concatenated outputs equal infer(cond, seed, window=24) of the finished frames' conditioning; a refused
    push in between changes nothing.  NVWN_FP32_FAST, which NVWaveNet does not create, runs the same session on its own engine
    against infer()'s window loop."""
    import torch
    from nv_wavenet_b200.nv_wavenet import Impl, LiveSession, NVWaveNet
    from nv_wavenet_b200.infer import live_ring_frames
    B = KINDS[kind][2]
    rng = np.random.default_rng(61)
    net = _network(rng)
    frames = rng.standard_normal((B, CC, 40)).astype(np.float32)
    lh = _host_batch(frames, net)
    w = refgen.lively_inputs(67, R, S, A, L, 1, 1)
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    for k, v in KINDS[kind][1].items():
        monkeypatch.setenv(k, v)
    fp16 = KINDS[kind][0] == "fp16"
    if kind == "fp32_fast":
        eng = _engine(kind, W, monkeypatch)
        eng.load(w)
        eng.cond_producer_open_live(*net, STRIDE, live_ring_frames(W, K, STRIDE))
        live = LiveSession(eng, CC, K, STRIDE, SEED, W)
        ref = _engine(kind, W, monkeypatch)
        ref.load(w)
        want = torch.empty((B, 200), dtype=torch.int32, device="cuda")
        NVWaveNet._generate(ref, torch.from_numpy(lh), None, SEED, None, want)
        want = want.cpu().numpy()
    else:
        wnet = _net(w, L, R, S, A, MD)
        live = wnet.open_live(*[torch.from_numpy(a) for a in net], STRIDE, B, SEED, window=W, fp16=fp16)
        cond = torch.from_numpy(np.ascontiguousarray(lh.transpose(3, 2, 1, 0))).cuda()
        want = wnet.infer(cond, Impl.AUTO, seed=SEED, fp16=fp16, window=W).cpu().numpy()
        assert wnet.engines_created == 1                                  # the session's engine is not infer()'s
    assert live.ring_frames == 8
    got, t = [], 0
    for i, n in enumerate([0, 1, 1, 4, 3, 15, 2, 14]):
        piece = frames[:, :, t:t + n]
        y = live.push(torch.from_numpy(piece).cuda() if i % 2 else piece)          # CUDA and host frames
        assert tuple(y.shape) == (B, n * STRIDE) and y.dtype == torch.int32 and y.is_cuda
        got.append(y.cpu().numpy())
        t += n
        assert live.frames == t and live.samples == t * STRIDE
        if i == 3:                                                        # 6 frames fit after frame 5: sample 30 reads frames 4 ..
            _refused(live._eng.cond_producer_push, np.zeros((B, CC, 7), np.float32),
                     match="nvwn_cond_producer_push: 7 frames would overwrite frame 4, which sample 30")
    got = np.concatenate(got, axis=1)
    assert np.array_equal(got, want), np.argwhere(got != want)[:5]
    assert len(np.unique(got)) > 8
    live.close()


def test_live_audio_option(monkeypatch):
    """push(audio=...) returns the samples' decoded audio, float and int16, as get_audio gives it for them."""
    import torch
    from nv_wavenet_b200 import _lib
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    rng = np.random.default_rng(71)
    net = _network(rng)
    frames = rng.standard_normal((3, CC, 9)).astype(np.float32)
    wnet = _net(refgen.lively_inputs(73, R, S, A, L, 1, 1), L, R, S, A, MD)
    lut = np.empty(A, np.float32)
    i16 = np.empty(A, np.int16)
    assert _lib.lib().nvwn_mulaw_table(A, C.c_void_p(lut.ctypes.data), C.c_void_p(i16.ctypes.data), None) == 0
    live = wnet.open_live(*net, STRIDE, 3, SEED, window=W, fp16=True)
    y, af = live.push(frames[:, :, :5], audio="float")
    y2, ai = live.push(frames[:, :, 5:], audio="int16")
    assert af.dtype == np.float32 and ai.dtype == np.int16 and af.shape == (3, 25) and ai.shape == (3, 20)
    assert np.array_equal(af, lut[y.cpu().numpy()]) and np.array_equal(ai, i16[y2.cpu().numpy()])
    live.close()


def _live_engine(N, monkeypatch, net, ring):
    """an fp32 engine of KINDS["fp32"]'s batch, its store zeroed, with a live sequence open"""
    e = _engine("fp32", N, monkeypatch)
    B = KINDS["fp32"][2]
    e.set_conditioning(np.zeros((N, L, B, 2 * R), np.float32), 0, N)
    e.cond_producer_open_live(*net, STRIDE, ring)
    return e


def test_ring_store_equals_loaded_store(monkeypatch):
    """The ring kernel: after each push and the productions it allows, the conditioning store equals the store a loaded producer of
    the finished frames writes for the same sample ranges, bit for bit."""
    B = KINDS["fp32"][2]
    rng = np.random.default_rng(79)
    net = _network(rng)
    frames = rng.standard_normal((B, CC, 30)).astype(np.float32)
    live = _live_engine(W, monkeypatch, net, 5)                          # 3 frames per push once the samples before them are produced
    loaded = _engine("fp32", W, monkeypatch)
    loaded.set_conditioning(np.zeros((W, L, B, 2 * R), np.float32), 0, W)
    loaded.cond_producer_load(frames, *net, STRIDE)
    t, done = 0, 0
    for n in [3, 1, 2, 3, 1, 3, 3, 2, 3, 3, 3, 3]:
        live.cond_producer_push(frames[:, :, t:t + n])
        t += n
        while done < t * STRIDE:                                          # pieces of at most 7 samples, across the store's wrap
            m = min(7, t * STRIDE - done)
            live.cond_producer_run_stream(done, m)
            loaded.cond_producer_run_stream(done, m)
            done += m
        live.synchronize()
        got, want = _store(live), _store(loaded)
        assert np.isfinite(got).all() and bits_equal(got, want), (t, np.argwhere(got.view(np.uint32) != want.view(np.uint32))[:5])
    assert t == 30 and np.abs(_store(live)).max() > 0.1


def test_refusals_change_nothing(monkeypatch):
    import nv_wavenet_b200 as nw
    from nv_wavenet_b200 import _lib
    lib = _lib.lib()
    B, N = KINDS["fp32"][2], W
    rng = np.random.default_rng(83)
    net = _network(rng)
    frames = rng.standard_normal((B, CC, 20)).astype(np.float32)
    e = _engine("fp32", N, monkeypatch)
    _refused(e.cond_producer_push, frames[:, :, :1], match="nvwn_cond_producer_push: no live sequence is open")
    _refused(e.cond_producer_open_live, *net, STRIDE, 3, match="nvwn_cond_producer_open_live: ring_frames = 3; need at least .* = 4")
    _refused(e.cond_producer_push, frames[:, :, :1], match="nvwn_cond_producer_push: no live sequence is open")
    e.cond_producer_open_live(*net, STRIDE, 4)
    _refused(e.cond_producer_open_live, *net, STRIDE, 3, match="ring_frames = 3")         # the open sequence stays open
    e.cond_producer_push(frames[:, :, :4])                               # a ring of 4 frames takes 4 before any production
    _refused(e.cond_producer_push, frames[:, :, 4:5], match="nvwn_cond_producer_push: 1 frames would overwrite frame 0, which sample 0")
    _refused(e.cond_producer_run_stream, 0, 21, match="nvwn_cond_producer_run_stream: samples \\[0, 21\\) of the live sequence are not all below the 20")
    _refused(e.cond_producer_run, 0, 0, 1, match="nvwn_cond_producer_run: a live sequence is produced with nvwn_cond_producer_run_stream")
    e.cond_producer_run_stream(0, 20)                                    # frame 4 is still not pushed; the refusals changed nothing
    e.cond_producer_run_stream(20, 0)
    e.cond_producer_push(frames[:, :, 4:6])                              # samples from 20 read frames 2 .. : 2 fit
    _refused(e.cond_producer_run_stream, 0, 5, match="nvwn_cond_producer_run_stream: frame 0, which sample 0 reads, has left the ring \\(it holds frames 2 .. 5\\)")
    _refused(e.cond_producer_run_stream, 16, 1, match="frame 1, which sample 16 reads, has left the ring")
    e.cond_producer_run_stream(17, 13)                                   # sample 17 reads frames 2 ..
    e.synchronize()
    got = _store(e)
    ref = _engine("fp32", N, monkeypatch)
    ref.cond_producer_load(frames[:, :, :6], *net, STRIDE)
    ref.cond_producer_run_stream(0, 20)
    ref.cond_producer_run_stream(17, 13)
    ref.synchronize()
    assert bits_equal(got, _store(ref))
    # nvwn_cond_producer_load ends the live sequence: pushes are refused, and run_stream follows the loaded sequence's rules
    e.cond_producer_load(frames[:, :, :2], *net, STRIDE)
    _refused(e.cond_producer_push, frames[:, :, 6:7], match="nvwn_cond_producer_push: no live sequence is open")
    _refused(e.cond_producer_run_stream, 0, 11, match="nvwn_cond_producer_run_stream: sample range outside num_frames \\* stride")
    e.cond_producer_run(0, 10)
    wu, bu, wc, bc = net
    p = lambda a: C.c_void_p(a.ctypes.data)
    for call in (lambda: lib.nvwn_cond_producer_push(e._h, p(frames), -1, None),
                 lambda: lib.nvwn_cond_producer_open_live(e._h, CC, p(wu), p(bu), 4, 5, p(wc), p(bc), 8, None)):    # window < stride
        with pytest.raises(nw.NvwnError, match="code -1"):
            _lib.check(call(), "live")
    e.synchronize()


def test_host_frames_may_be_reused_on_return(monkeypatch):
    """Frames in pinned host memory, overwritten as soon as each push returns, leave the store that ordinary arrays leave."""
    import torch
    B = KINDS["fp32"][2]
    rng = np.random.default_rng(89)
    net = _network(rng)
    frames = rng.standard_normal((B, CC, 8)).astype(np.float32)
    stores = []
    for pinned in (False, True):
        e = _live_engine(2 * W, monkeypatch, net, 8)
        for a, b in ((0, 3), (3, 8)):
            if pinned:
                f = torch.from_numpy(np.ascontiguousarray(frames[:, :, a:b])).pin_memory()
                e.cond_producer_push(f)
                f.fill_(1e6)
            else:
                e.cond_producer_push(frames[:, :, a:b])
            e.cond_producer_run_stream(a * STRIDE, (b - a) * STRIDE)
        torch.cuda.synchronize()
        stores.append(_store(e))
    assert bits_equal(stores[0], stores[1]) and np.abs(stores[0]).max() > 0.1
