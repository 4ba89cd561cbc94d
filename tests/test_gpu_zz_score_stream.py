"""Streaming scoring (nvwn_score_stream): an engine of W samples whose conditioning store is a ring scores audio of any length, a
window at a time, bit-identically to nvwn_score of one engine that holds the whole length -- logp and logits -- on every engine
kind, from expanded conditioning and from mel frames, without touching the generation state."""
import ctypes as C

import numpy as np
import pytest
import torch

import nv_wavenet_b200 as nw
from nv_wavenet_b200 import _lib
from tests import refgen
from tests.common import bits_equal

pytestmark = pytest.mark.gpu

EINVAL, EUNSUPPORTED = -1, -2
R, S, A = 64, 256, 256
L, MD = 14, 64                        # dilations 1 .. 64 twice: the fronts of most layers are longer than short calls
KINDS = {"lat": nw.KERNEL_LATENCY, "tc": nw.KERNEL_TENSORCORE, "stream": nw.KERNEL_STREAM}
LAUNCH_KERNEL = {"lat": 18, "tc": 17, "stream": 16}


def _engine(w, B, N, kind="lat", Lm=L, md=MD):
    e = nw.NVWavenetInfer(Lm, md, B, N, KINDS[kind], True, R=R, S=S, A=A, dtype=nw.FP16)
    e.load(w)
    return e


def _ranges(total, W):
    """Uneven calls of at most W samples: some of exactly W, some of 1 and 2, most not dividing W, many crossing the wrap."""
    sizes = [W, max(1, W - 2), 1, W, (W + 1) // 2, 2]
    out, first, i = [], 0, 0
    while first < total:
        n = min(sizes[i % len(sizes)], total - first)
        out.append((first, n))
        first += n; i += 1
    return out


def _whole(w, lh, audio, kind="lat"):
    """nvwn_score of one engine that holds the whole length: (logp, logits)."""
    B, T = audio.shape
    e = _engine(w, B, T, kind)
    e.set_conditioning(lh, 0, T)
    out = e.score(audio, logits=True)
    e.close()
    return out


def _streamed(e, lh, audio, ranges, logits=True):
    """score_stream over `ranges`, each call's conditioning put in the ring just before it: (logp, logits)."""
    B, T = audio.shape
    lp = np.full((B, T), np.nan, np.float32)
    lg = np.full((B, T, A), np.nan, np.float32) if logits else None
    for first, n in ranges:
        e.set_conditioning_stream(lh[first:first + n], first)
        got = e.score_stream(audio[:, first:first + n], first, logits=logits)
        if logits:
            lp[:, first:first + n], lg[:, first:first + n] = got
        else:
            lp[:, first:first + n] = got
    return lp, lg


def _inputs(seed, B, T):
    w = refgen.lively_inputs(seed, R, S, A, L, 1, 1)
    rng = np.random.default_rng(seed)
    lh = (0.5 * rng.standard_normal((T, L, B, 2 * R))).astype(np.float32)
    audio = rng.integers(0, A, (B, T)).astype(np.int32)
    return w, lh, audio


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_window_invariance(kind):
    """W in {7, 50, 64, 100, 256} over 700 samples (several wraps of every ring), calls of uneven counts; the three kinds agree."""
    B, T = 8, 700
    w, lh, audio = _inputs(21, B, T)
    ref = _whole(w, lh, audio, "lat")
    own = _whole(w, lh, audio, kind) if kind != "lat" else ref
    assert np.isfinite(ref[1]).all() and (ref[0] <= 0).all()
    assert bits_equal(ref[0], own[0]) and bits_equal(ref[1], own[1]), f"{kind}: nvwn_score differs from the latency engine's"
    for W in (7, 50, 64, 100, 256):
        e = _engine(w, B, W, kind)
        lp, lg = _streamed(e, lh, audio, _ranges(T, W))
        assert bits_equal(own[0], lp), f"W = {W}: logp differs at {np.argwhere(own[0].view(np.uint32) != lp.view(np.uint32))[:3]}"
        assert bits_equal(own[1], lg), f"W = {W}: logits differ"
        e.close()


def test_window_larger_than_the_scorer_chunk():
    """B = 128: the scorer's time chunk is 16384 / 128 = 128 steps, so a call of W = 256 samples runs in two chunks and a call's
    fronts come both from its own chunks and from the previous call."""
    B, T, W = 128, 700, 256
    w, lh, audio = _inputs(22, B, T)
    ref = _whole(w, lh, audio)
    e = _engine(w, B, W)
    lp, lg = _streamed(e, lh, audio, _ranges(T, W))
    assert bits_equal(ref[0], lp) and bits_equal(ref[1], lg)


def test_fresh_restart():
    """A new stream at first_sample = 0, after a whole stream and after one broken off, gives the first pass's bits."""
    B, T, W = 5, 300, 50
    w, lh, audio = _inputs(23, B, T)
    e = _engine(w, B, W)
    first = _streamed(e, lh, audio, _ranges(T, W))
    again = _streamed(e, lh, audio, _ranges(T, W))
    assert bits_equal(first[0], again[0]) and bits_equal(first[1], again[1])
    other = np.random.default_rng(5).integers(0, A, (B, T)).astype(np.int32)
    _streamed(e, lh, other, _ranges(130, W))                            # broken off after 130 samples of other audio
    third = _streamed(e, lh, audio, _ranges(T, W))
    assert bits_equal(first[0], third[0]) and bits_equal(first[1], third[1])


def test_independent_of_generation():
    """Streaming generation, reset_history and restart_slots between score_stream calls on one engine: the scores equal those of
    the whole-length engine, and every generation window's samples, dumps and launch info equal an engine that never scored."""
    B, W, windows = 8, 64, 6
    T = W * windows
    w, lh, audio = _inputs(24, B, T)
    ref = _whole(w, lh, audio)
    seed = 0x5C0DE
    gen_lh = (0.5 * np.random.default_rng(25).standard_normal((T, L, B, 2 * R))).astype(np.float32)

    def generation(e, k, state, score=None):
        if score is not None:
            score(k)
        if k == 2:
            e.reset_history()
            state["first"] = 0
        if k == 4:
            e.restart_slots([1, 6], [11, 12])
        first = state["first"]
        n = W - 3 if k % 2 else W
        e.set_conditioning_stream(gen_lh[first:first + n], first)
        e.set_selectors_random_stream(seed, first, n)
        e.run_stream(first, n, B, dump_activations=True)
        y = np.zeros((B, n), np.int32)
        e.get_yout_stream(y, first, n)
        e.synchronize()
        state["first"] = first + n
        return y, e.activations(), e.launch_info()

    plain = _engine(w, B, W)
    plain.reset_history()
    st = {"first": 0}
    expect = [generation(plain, k, st) for k in range(windows)]

    e = _engine(w, B, W)
    e.reset_history()
    lp = np.full((B, T), np.nan, np.float32)
    lg = np.full((B, T, A), np.nan, np.float32)

    def score(k):
        first = k * W
        e.set_conditioning_stream(lh[first:first + W], first)
        lp[:, first:first + W], lg[:, first:first + W] = e.score_stream(audio[:, first:first + W], first, logits=True)

    st = {"first": 0}
    for k in range(windows):
        y, acts, info = generation(e, k, st, score)
        ye, acts_e, info_e = expect[k]
        assert np.array_equal(y, ye), f"window {k}: samples differ"
        for name in acts:
            assert bits_equal(acts[name], acts_e[name]), f"window {k}: the {name} dump differs"
        assert info == info_e, f"window {k}: launch info differs"
    assert info["kernel"] == LAUNCH_KERNEL["lat"]
    assert bits_equal(ref[0], lp) and bits_equal(ref[1], lg)


def _rc(e, audio, first, count, bs, logp, logits=None):
    lib = _lib.lib()
    ptr = lambda a: None if a is None else C.c_void_p(a.ctypes.data)
    code = lib.nvwn_score_stream(None if e is None else e._h, ptr(audio), first, count, bs, ptr(logp), ptr(logits), None)
    return code, lib.nvwn_last_error().decode()


def test_ending_and_errors():
    B, W, T, Lm, md = 3, 12, 40, 4, 4
    w = refgen.lively_inputs(26, R, S, A, Lm, 1, 1)
    rng = np.random.default_rng(26)
    lh = (0.5 * rng.standard_normal((T, Lm, B, 2 * R))).astype(np.float32)
    audio = rng.integers(0, A, (B, T)).astype(np.int32)
    e = _engine(w, B, W, Lm=Lm, md=md)
    whole = _engine(w, B, T, Lm=Lm, md=md)
    whole.set_conditioning(lh, 0, T)
    ref = whole.score(audio)
    ranges = [(0, 12), (12, 12), (24, 12), (36, 4)]

    def call(k, bs=B):
        first, n = ranges[k]
        e.set_conditioning_stream(lh[first:first + n], first)
        a = np.ascontiguousarray(audio[:bs, first:first + n])
        lp = np.empty((bs, n), np.float32)
        code, msg = _rc(e, a, first, n, bs, lp)
        return code, msg, lp

    def restart_and_check():
        for k in range(len(ranges)):
            code, msg, lp = call(k)
            assert code == 0, msg
            first, n = ranges[k]
            assert bits_equal(ref[:, first:first + n], lp), f"call {k}"

    # nvwn_score and every kind of weight change end the stream
    enders = {"nvwn_score": lambda: e.score(audio[:, :W]),
              "set_layer_weights": lambda: e.set_layer_weights(1, w["Wprev"][1], w["Wcur"][1], w["Bh"][1], w["Wres"][1], w["Bres"][1],
                                                               w["Wskip"][1], w["Bskip"][1]),
              "set_out_weights": lambda: e.set_out_weights(w["Wzs"], w["Bzs"], w["Wza"], w["Bza"]),
              "set_embeddings": lambda: e.set_embeddings(w["embPrev"], w["embCur"]),
              "weights_updated": lambda: e.weights_updated()}
    for name, end in enders.items():
        assert call(0)[0] == 0 and call(1)[0] == 0
        end()
        code, msg, _ = call(2)
        assert code == EINVAL and "first_sample = 0" in msg, f"{name}: {code} {msg}"
        restart_and_check()

    # argument checks: each EINVAL names what is wrong and leaves the stream as it was
    assert call(0)[0] == 0
    a, lp = np.ascontiguousarray(audio[:, 12:24]), np.empty((B, 12), np.float32)
    assert _rc(None, a, 12, 12, B, lp)[0] == EINVAL
    assert _rc(e, None, 12, 12, B, lp)[0] == EINVAL
    code, msg = _rc(e, a, 12, 12, B, None)
    assert code == EINVAL and "nvwn_score_stream" in msg
    for n in (0, W + 1):
        code, msg = _rc(e, np.zeros((B, W + 1), np.int32), 12, n, B, np.empty((B, W + 1), np.float32))
        assert code == EINVAL and "count" in msg, msg
    code, msg = _rc(e, a, -12, 12, B, lp)
    assert code == EINVAL and "first_sample" in msg and "< 0" in msg, msg
    code, msg = _rc(e, a, 13, 12, B, lp)
    assert code == EINVAL and "the next sample is 12" in msg, msg
    for bs in (0, B + 1):
        code, msg = _rc(e, a, 12, 12, bs, lp)
        assert code == EINVAL and "batch_size" in msg, msg
    code, msg = _rc(e, a, 12, 12, B - 1, lp)
    assert code == EINVAL and "batch_size 2" in msg and "batch_size 3" in msg, msg
    bad = a.copy(); bad[1, 7] = A; bad[2, 3] = -1
    code, msg = _rc(e, bad, 12, 12, B, lp)
    assert code == EINVAL and "audio[1][19]" in msg, msg                  # absolute t = 12 + 7
    with pytest.raises(nw.NvwnError, match=r"audio\[1\]\[19\]"):
        e.score_stream(torch.from_numpy(bad).cuda(), 12)
    for k in (1, 2, 3):                                                  # the stream goes on from 12 as if nothing had happened
        code, msg, got = call(k)
        first, n = ranges[k]
        assert code == 0 and bits_equal(ref[:, first:first + n], got), msg

    # a batch_size below B is a stream of its own, and a new stream may change it
    for k in range(len(ranges)):
        code, msg, got = call(k, bs=2)
        first, n = ranges[k]
        assert code == 0 and bits_equal(ref[:2, first:first + n], got), msg

    e32 = nw.NVWavenetInfer(Lm, md, B, W, R=R, S=S, A=A, dtype=nw.FP32)
    code, msg = _rc(e32, a, 0, 12, B, lp)
    assert code == EUNSUPPORTED and "FP16" in msg and "nvwn_score_stream" in msg
    e512 = nw.NVWavenetInfer(Lm, md, 1, 4, R=R, S=S, A=512, dtype=nw.FP16)
    code, msg = _rc(e512, a, 0, 4, 1, lp)
    assert code == EUNSUPPORTED and "A = 256" in msg


def _c3_frames(B, frames, seed=27):
    """C3 model and an 80-channel mel front end of window 800, stride 200: weights, features [B][80][frames], network."""
    Lc, Cc, K, stride = 20, 80, 800, 200
    w = refgen.lively_inputs(seed, R, S, A, Lc, 1, 1)
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s, sc=1.0: sc * torch.randn(s, generator=g, device="cuda")
    features = rn(B, Cc, frames)
    net = (rn(Cc, Cc, K, sc=1 / np.sqrt(Cc * K / stride)), rn(Cc, sc=0.1), rn(Lc * 2 * R, Cc, sc=0.5 / np.sqrt(Cc)), rn(Lc * 2 * R, sc=0.1))
    return w, features, net, stride


def test_c3_from_frames():
    """64 x (3 * 16 000 + 200) samples through W = 4096, each window's conditioning made by cond_producer_run_stream, against one
    engine of the whole length filled by set_conditioning_from_features and scored by nvwn_score."""
    B, W, frames = 64, 4096, (3 * 16000 + 200) // 200
    w, features, net, stride = _c3_frames(B, frames)
    T = frames * stride
    audio = torch.randint(0, A, (B, T), generator=torch.Generator(device="cuda").manual_seed(28), device="cuda", dtype=torch.int32)
    whole = nw.NVWavenetInfer(20, 512, B, T, R=R, S=S, A=A, dtype=nw.FP16)
    whole.load(w)
    whole.set_conditioning_from_features(features, *net, stride)
    lp_ref, lg_ref = whole.score(audio, logits=True)
    torch.cuda.synchronize()
    whole.close()
    del whole

    e = nw.NVWavenetInfer(20, 512, B, W, R=R, S=S, A=A, dtype=nw.FP16)
    e.load(w)
    e.cond_producer_load(features, *net, stride)
    lp = torch.empty_like(lp_ref)
    for first in range(0, T, W):
        n = min(W, T - first)
        e.cond_producer_run_stream(first, n)
        got_lp, got_lg = e.score_stream(audio[:, first:first + n], first, logits=True)
        lp[:, first:first + n] = got_lp
        assert torch.equal(got_lg.view(torch.int32), lg_ref[:, first:first + n].view(torch.int32)), f"logits differ in the window at {first}"
        del got_lg
    torch.cuda.synchronize()
    assert torch.isfinite(lp_ref).all()
    assert torch.equal(lp.view(torch.int32), lp_ref.view(torch.int32))


def _small_net(seed):
    from nv_wavenet_b200.nv_wavenet import NVWaveNet
    g = torch.Generator().manual_seed(seed)
    n = lambda *shape, s=0.5: (s * torch.randn(*shape, generator=g)).cuda()
    Lm = 6
    kw = dict(embedding_prev=n(A, R), embedding_curr=n(A, R), conv_out_weight=n(A, S, s=1 / 16), conv_end_weight=n(A, A, s=1 / 8),
              dilate_weights=[n(2 * R, R, 2, s=0.1) for _ in range(Lm)], dilate_biases=[n(2 * R, s=0.1) for _ in range(Lm)],
              max_dilation=16, res_weights=[n(R, R, s=0.1) for _ in range(Lm - 1)], res_biases=[n(R, s=0.05) for _ in range(Lm - 1)],
              skip_weights=[n(S, R, s=0.1) for _ in range(Lm)], skip_biases=[n(S, s=0.05) for _ in range(Lm)], use_embed_tanh=True)
    return NVWaveNet(**kw), Lm, g


def test_nvwavenet_log_likelihood_windows():
    net, Lm, g = _small_net(29)
    Bn, Nn = 3, 250
    cond = (0.5 * torch.randn(2 * R, Bn, Lm, Nn, generator=g)).cuda()
    aud = torch.randint(0, A, (Bn, Nn), generator=g).to(torch.int32)
    whole = net.log_likelihood(cond, aud)
    for W in (7, 64, 100, 250, 300):
        for a in (aud, aud.cuda()):                                      # host and device audio
            got = net.log_likelihood(cond, a, window=W)
            assert got.is_cuda and tuple(got.shape) == (Bn, Nn)
            assert bits_equal(whole.cpu().numpy(), got.cpu().numpy()), f"W = {W}"


def test_nvwavenet_log_likelihood_from_features():
    net, Lm, g = _small_net(30)
    Bn, Cc, frames, K, stride = 3, 7, 24, 12, 5
    rng = np.random.default_rng(30)
    features = rng.standard_normal((Bn, Cc, frames)).astype(np.float32)
    wu = (rng.standard_normal((Cc, Cc, K)) / np.sqrt(Cc * K / stride)).astype(np.float32)
    bu = (0.1 * rng.standard_normal(Cc)).astype(np.float32)
    wc = (0.5 * rng.standard_normal((Lm * 2 * R, Cc, 1)) / np.sqrt(Cc)).astype(np.float32)
    bc = (0.1 * rng.standard_normal(Lm * 2 * R)).astype(np.float32)
    T = frames * stride
    audio = rng.integers(0, A, (Bn, T)).astype(np.int32)
    lh = np.full((T, Lm, Bn, 2 * R), np.nan, np.float32)
    p = lambda a: C.c_void_p(np.ascontiguousarray(a, np.float32).ctypes.data)
    f = np.ascontiguousarray(features)
    assert _lib.lib().nvwn_cond_from_features_host(p(lh), C.c_void_p(f.ctypes.data), Bn, Cc, frames, p(wu), p(bu), K, stride,
                                                    p(wc), p(bc), Lm, R) == 0
    ref = net.log_likelihood(torch.from_numpy(lh).permute(3, 2, 1, 0), torch.from_numpy(audio)).cpu().numpy()
    whole = net.log_likelihood_from_features(features, audio, wu, bu, wc, bc, stride).cpu().numpy()
    assert bits_equal(ref, whole)
    timing = {}
    for W in (9, 64, T):
        got = net.log_likelihood_from_features(features, audio, wu, bu, wc, bc, stride, window=W, timing=timing)
        assert bits_equal(ref, got.cpu().numpy()), f"W = {W}"
        assert timing["produce_s"] > 0 and timing["score_s"] > 0
    dev = lambda a: torch.from_numpy(a).cuda()                           # device frames, network and audio
    got = net.log_likelihood_from_features(dev(features), dev(audio), dev(wu), dev(bu), dev(wc), dev(bc), stride, window=64)
    assert bits_equal(ref, got.cpu().numpy())


def test_side_stream_device_outputs():
    """CUDA audio and outputs on a side stream equal host arrays on the default stream."""
    B, T, W = 4, 200, 64
    w, lh, audio = _inputs(31, B, T)
    e = _engine(w, B, W)
    host = _streamed(e, lh, audio, _ranges(T, W))
    s = torch.cuda.Stream()
    d_audio = torch.from_numpy(audio).cuda()
    lp = torch.empty((B, T), device="cuda")
    lg = torch.empty((B, T, A), device="cuda")
    for first, n in _ranges(T, W):
        s.synchronize()
        e.set_conditioning_stream(lh[first:first + n], first)
        with torch.cuda.stream(s):
            a = d_audio[:, first:first + n].contiguous()
            got_lp, got_lg = e.score_stream(a, first, logits=True, stream=s)
            assert got_lp.is_cuda and got_lg.is_cuda
            lp[:, first:first + n] = got_lp
            lg[:, first:first + n] = got_lg
    s.synchronize()
    assert bits_equal(host[0], lp.cpu().numpy()) and bits_equal(host[1], lg.cpu().numpy())
