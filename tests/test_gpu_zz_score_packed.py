"""Packed scoring (nvwn_score_stream_packed): utterances placed end to end in the rows of one scoring stream, each one's logp and
logits bit-identical to nvwn_score of it alone, on every engine kind, whatever the calls, windows and scorer chunks; the stream's
calling rules; and the queue calls NVWaveNet.log_likelihood_many and log_likelihood_many_from_features."""
import ctypes as C

import numpy as np
import pytest
import torch

import nv_wavenet_b200 as nw
from nv_wavenet_b200 import _lib
from tests import refgen
from tests.common import bits_equal
from tests.test_gpu_zz_score_stream import LAUNCH_KERNEL, MD, A, L, R, S, _engine, _ranges, _small_net

pytestmark = pytest.mark.gpu

EINVAL, EUNSUPPORTED = -1, -2


def _rows(B, T, W, seed):
    """Per row the sorted utterance starts in [0, T), row 0 always starting at 0, chosen so that starts fall at a call's first and
    last sample (calls _ranges(T, W)), in mid-chunk and on both sides of a scorer-chunk boundary (chunks of 16384 / B steps), within
    d_l of the previous start for small and large d_l, and on utterances of 1, 2, MD - 1, MD and MD + 1 samples; one row holds a
    single utterance longer than several windows."""
    rng = np.random.default_rng(seed)
    calls = _ranges(T, W)
    chunk = 16384 // B
    cum = lambda gaps: sorted({0} | {int(v) for v in np.cumsum(gaps) if v < T})
    rows = [cum([1, 2, MD - 1, MD, MD + 1, 1, 1, 2, MD + 1, MD - 1, MD]),          # utterances of 1, 2, MD - 1, MD, MD + 1 samples
            cum([3, 1, 2, 5, 33, 7, 60, 1, 4, 100, 16, 8, 31]),                    # starts within d_l of the last for small and large d_l
            [0],                                                                   # one utterance of every sample
            sorted({0} | {f for f, n in calls[2:9]} | {f + n - 1 for f, n in calls[3:10]}),   # a call's first and last sample
            sorted({0} | {f + k for f, n in calls for k in (chunk - 1, chunk, chunk + 1, chunk // 2) if k < n})]  # chunk edges
    while len(rows) < B:
        rows.append(cum(rng.integers(1, 160, 20)))
    return rows[:B]


def _queue(rows, T, seed):
    """The stream [T] of each row's utterances and the utterances: audio [B][T], starts [B][T], lh [T][L][B][2R] and per utterance
    (row, start, length)."""
    B = len(rows)
    rng = np.random.default_rng(seed)
    audio = rng.integers(0, A, (B, T)).astype(np.int32)
    lh = (0.5 * rng.standard_normal((T, L, B, 2 * R))).astype(np.float32)
    starts = np.zeros((B, T), np.uint8)
    utts = []
    for b, st in enumerate(rows):
        starts[b, st] = 1
        ends = st[1:] + [T]
        utts += [(b, s, e - s) for s, e in zip(st, ends)]
    return audio, starts, lh, utts


_ALONE = {}


def _alone(w, audio, lh, utts, key):
    """nvwn_score of every utterance alone, in one one-utterance engine: (logp [n], logits [n][A]) per utterance."""
    if key not in _ALONE:
        T = audio.shape[1]
        e = _engine(w, 1, T)
        out = []
        for b, s, n in utts:
            e.set_conditioning(np.ascontiguousarray(lh[s:s + n, :, b:b + 1]), 0, n)
            lp, lg = e.score(np.ascontiguousarray(audio[b:b + 1, s:s + n]), logits=True)
            out.append((lp[0], lg[0]))
        e.close()
        _ALONE[key] = out
    return _ALONE[key]


def _packed(e, audio, starts, lh, ranges, packed=True):
    """score_stream_packed (or score_stream) over `ranges`, each call's conditioning put in the ring just before it."""
    B, T = audio.shape
    lp = np.full((B, T), np.nan, np.float32)
    lg = np.full((B, T, A), np.nan, np.float32)
    for first, n in ranges:
        e.set_conditioning_stream(lh[first:first + n], first)
        a = audio[:, first:first + n]
        got = e.score_stream_packed(a, starts[:, first:first + n], first, logits=True) if packed else e.score_stream(a, first, logits=True)
        lp[:, first:first + n], lg[:, first:first + n] = got
    return lp, lg


def _check_alone(lp, lg, utts, alone, what):
    for (b, s, n), (rp, rg) in zip(utts, alone):
        assert bits_equal(rp, lp[b, s:s + n]), f"{what}: logp of the utterance of row {b} at {s} ({n} samples) differs from it alone"
        assert bits_equal(rg, lg[b, s:s + n]), f"{what}: logits of the utterance of row {b} at {s} ({n} samples) differ from it alone"


@pytest.mark.parametrize("kind,B,W", [("lat", 8, 64), ("tc", 8, 64), ("stream", 8, 64), ("lat", 128, 256)])
def test_packed_equals_alone(kind, B, W):
    """Every utterance of the packed rows gives the bits of nvwn_score of it alone, through uneven calls that cross the store's
    wrap; B = 128 makes the scorer's chunk 128 steps, so calls of W = 256 run in two chunks."""
    T = 700
    w = refgen.lively_inputs(41, R, S, A, L, 1, 1)
    rows = _rows(B, T, W, 42)
    audio, starts, lh, utts = _queue(rows, T, 43 + B)
    alone = _alone(w, audio, lh, utts, (B, W))
    e = _engine(w, B, W, kind)
    lp, lg = _packed(e, audio, starts, lh, _ranges(T, W))
    assert np.isfinite(lg).all()
    _check_alone(lp, lg, utts, alone, f"{kind}, B = {B}, W = {W}")
    e.close()


def test_starts_only_at_zero_equal_score_stream():
    B, T, W = 8, 500, 64
    w = refgen.lively_inputs(44, R, S, A, L, 1, 1)
    audio, starts, lh, _ = _queue([[0]] * B, T, 45)
    starts[:, 0] = 0                                                        # every row starts at sample 0 whatever the flags say
    e = _engine(w, B, W)
    plain = _packed(e, audio, starts, lh, _ranges(T, W), packed=False)
    packed = _packed(e, audio, starts, lh, _ranges(T, W))
    assert bits_equal(plain[0], packed[0]) and bits_equal(plain[1], packed[1])


def test_window_invariance():
    B, T = 6, 400
    w = refgen.lively_inputs(46, R, S, A, L, 1, 1)
    audio, starts, lh, utts = _queue(_rows(B, T, 50, 47), T, 48)
    ref = None
    for W in (1, 2, 7, 50, 64, 400):
        e = _engine(w, B, W)
        calls = _ranges(T, W) if W > 2 else [(f, min(W, T - f)) for f in range(0, T, W)]      # _ranges has calls of 2 samples
        got = _packed(e, audio, starts, lh, calls)
        e.close()
        if ref is None:
            ref = got
            _check_alone(got[0], got[1], utts, _alone(w, audio, lh, utts, ("inv", B)), f"W = {W}")
        assert bits_equal(ref[0], got[0]) and bits_equal(ref[1], got[1]), f"W = {W} differs from W = 1"


def _rc(fn, e, audio, starts, first, count, bs, logp):
    lib = _lib.lib()
    ptr = lambda a: None if a is None else C.c_void_p(a.ctypes.data)
    h = None if e is None else e._h
    code = (lib.nvwn_score_stream_packed(h, ptr(audio), ptr(starts), first, count, bs, ptr(logp), None, None) if fn == "packed"
            else lib.nvwn_score_stream(h, ptr(audio), first, count, bs, ptr(logp), None, None))
    return code, lib.nvwn_last_error().decode()


def test_rules():
    B, W, T, Lm, md = 3, 12, 48, 4, 4
    w = refgen.lively_inputs(49, R, S, A, Lm, 1, 1)
    rng = np.random.default_rng(49)
    lh = (0.5 * rng.standard_normal((T, Lm, B, 2 * R))).astype(np.float32)
    audio = rng.integers(0, A, (B, T)).astype(np.int32)
    starts = np.zeros((B, T), np.uint8)
    starts[0, [5, 12, 13, 30]] = 1; starts[1, [2, 23, 24]] = 1; starts[2, 40] = 1
    ranges = [(0, 12), (12, 12), (24, 12), (36, 12)]

    def call(e, k, fn="packed", a=None):
        first, n = ranges[k]
        e.set_conditioning_stream(lh[first:first + n], first)
        a = np.ascontiguousarray(audio[:, first:first + n] if a is None else a)
        lp = np.empty((B, n), np.float32)
        code, msg = _rc(fn, e, a, np.ascontiguousarray(starts[:, first:first + n]), first, n, B, lp)
        return code, msg, lp

    clean = _engine(w, B, W, Lm=Lm, md=md)
    ref = np.concatenate([call(clean, k)[2] for k in range(4)], axis=1)
    e = _engine(w, B, W, Lm=Lm, md=md)

    # a stream is packed or not from its first call
    assert call(e, 0)[0] == 0
    code, msg, _ = call(e, 1, "plain")
    assert code == EINVAL and "packed" in msg and "nvwn_score_stream_packed" in msg, msg
    assert call(e, 0, "plain")[0] == 0
    code, msg, _ = call(e, 1)
    assert code == EINVAL and "not packed" in msg, msg

    # primes refuse a packed stream
    assert call(e, 0)[0] == 0
    with pytest.raises(nw.NvwnError, match="packed"):
        e.prime_from_score()
    with pytest.raises(nw.NvwnError, match="packed"):
        e.prime_slots_from_score([0], [1])
    for k in (1, 2, 3):                                                  # and leave it as it was
        code, msg, got = call(e, k)
        assert code == 0 and bits_equal(ref[:, 12 * k:12 * k + 12], got), msg

    # a weight change ends it
    assert call(e, 0)[0] == 0
    e.set_out_weights(w["Wzs"], w["Bzs"], w["Wza"], w["Bza"])
    code, msg, _ = call(e, 1)
    assert code == EINVAL and "first_sample = 0" in msg, msg

    # starts NULL
    lp = np.empty((B, 12), np.float32)
    code, msg = _rc("packed", e, np.ascontiguousarray(audio[:, :12]), None, 0, 12, B, lp)
    assert code == EINVAL and "starts" in msg, msg

    # a bad audio value is refused, and the stream goes on as if the call had never been made
    assert call(e, 0)[0] == 0 and call(e, 1)[0] == 0
    bad = audio[:, 24:36].copy(); bad[2, 4] = A
    code, msg, _ = call(e, 2, a=bad)
    assert code == EINVAL and "audio[2][28]" in msg, msg
    for k in (2, 3):
        code, msg, got = call(e, k)
        assert code == 0 and bits_equal(ref[:, 12 * k:12 * k + 12], got), msg


def test_independent_of_generation():
    """Streaming generation, reset_history and restart_slots between packed scoring calls on one engine: the scores equal those of
    an engine that only scored, and every generation window equals an engine that never scored."""
    B, W, windows = 8, 64, 6
    T = W * windows
    w = refgen.lively_inputs(50, R, S, A, L, 1, 1)
    audio, starts, lh, _ = _queue(_rows(B, T, W, 51), T, 52)
    calls = [(k * W, W) for k in range(windows)]
    ref = _packed(_engine(w, B, W), audio, starts, lh, calls)
    seed = 0x5C0DE
    gen_lh = (0.5 * np.random.default_rng(53).standard_normal((T, L, B, 2 * R))).astype(np.float32)

    def generation(e, k, state):
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
    st = {"first": 0}
    for k in range(windows):
        first = k * W
        e.set_conditioning_stream(lh[first:first + W], first)
        lp[:, first:first + W], lg[:, first:first + W] = e.score_stream_packed(audio[:, first:first + W], starts[:, first:first + W], first,
                                                                               logits=True)
        y, acts, info = generation(e, k, st)
        ye, acts_e, info_e = expect[k]
        assert np.array_equal(y, ye), f"window {k}: samples differ"
        for name in acts:
            assert bits_equal(acts[name], acts_e[name]), f"window {k}: the {name} dump differs"
        assert info == info_e, f"window {k}: launch info differs"
    assert info["kernel"] == LAUNCH_KERNEL["lat"]
    assert bits_equal(ref[0], lp) and bits_equal(ref[1], lg)


def test_device_starts_on_a_side_stream():
    """CUDA audio and start flags on a side stream equal host arrays."""
    B, T, W = 5, 200, 64
    w = refgen.lively_inputs(54, R, S, A, L, 1, 1)
    audio, starts, lh, _ = _queue(_rows(B, T, W, 55), T, 56)
    e = _engine(w, B, W)
    host = _packed(e, audio, starts, lh, _ranges(T, W))
    s = torch.cuda.Stream()
    lp = torch.empty((B, T), device="cuda")
    for first, n in _ranges(T, W):
        s.synchronize()
        e.set_conditioning_stream(lh[first:first + n], first)
        with torch.cuda.stream(s):
            a = torch.from_numpy(audio[:, first:first + n].copy()).cuda()
            f = torch.from_numpy(starts[:, first:first + n].copy()).cuda()
            got = e.score_stream_packed(a, f, first, stream=s)
            assert got.is_cuda
            lp[:, first:first + n] = got
    s.synchronize()
    assert bits_equal(host[0], lp.cpu().numpy())


def test_log_likelihood_many():
    net, Lm, g = _small_net(57)
    rng = np.random.default_rng(57)
    lengths = [int(v) for v in rng.integers(1, 90, 11)] + [1, 2, 17, 250]
    conds = [(0.5 * torch.randn(2 * R, Lm, n, generator=g)).cuda() for n in lengths]
    auds = [torch.randint(0, A, (n,), generator=g).to(torch.int32) for n in lengths]
    ref = [net.log_likelihood(c[:, None], a[None])[0] for c, a in zip(conds, auds)]
    timing = {}
    for slots, W in ((4, 50), (3, 7), (16, 64)):
        got = net.log_likelihood_many(conds, auds, slots=slots, window=W, timing=timing)
        assert len(got) == len(lengths) and timing["produce_s"] > 0 and timing["score_s"] > 0
        for u, (r, o) in enumerate(zip(ref, got)):
            assert o.is_cuda and o.dtype == torch.float32 and tuple(o.shape) == (lengths[u],)
            assert bits_equal(r.cpu().numpy(), o.cpu().numpy()), f"slots = {slots}, W = {W}: utterance {u} differs from it alone"


def test_log_likelihood_many_from_features():
    net, Lm, g = _small_net(58)
    rng = np.random.default_rng(58)
    Cc, K, stride = 7, 12, 5
    frames = [int(v) for v in rng.integers(1, 20, 9)]
    features = [rng.standard_normal((Cc, n)).astype(np.float32) for n in frames]
    wu = (rng.standard_normal((Cc, Cc, K)) / np.sqrt(Cc * K / stride)).astype(np.float32)
    bu = (0.1 * rng.standard_normal(Cc)).astype(np.float32)
    wc = (0.5 * rng.standard_normal((Lm * 2 * R, Cc, 1)) / np.sqrt(Cc)).astype(np.float32)
    bc = (0.1 * rng.standard_normal(Lm * 2 * R)).astype(np.float32)
    auds = [rng.integers(0, A, n * stride).astype(np.int32) for n in frames]
    p = lambda a: C.c_void_p(np.ascontiguousarray(a, np.float32).ctypes.data)
    ref = []
    for f, a in zip(features, auds):
        n = f.shape[1] * stride
        lh = np.full((n, Lm, 1, 2 * R), np.nan, np.float32)
        f = np.ascontiguousarray(f)
        assert _lib.lib().nvwn_cond_from_features_host(p(lh), C.c_void_p(f.ctypes.data), 1, Cc, f.shape[1], p(wu), p(bu), K, stride, p(wc),
                                                        p(bc), Lm, R) == 0
        ref.append(net.log_likelihood(torch.from_numpy(lh).permute(3, 2, 1, 0), torch.from_numpy(a)[None])[0].cpu().numpy())
    timing = {}
    for slots, W in ((3, 32), (4, 9)):
        got = net.log_likelihood_many_from_features(features, auds, wu, bu, wc, bc, stride, slots=slots, window=W, timing=timing)
        assert timing["produce_s"] > 0 and timing["score_s"] > 0
        for u, (r, o) in enumerate(zip(ref, got)):
            assert bits_equal(r, o.cpu().numpy()), f"slots = {slots}, W = {W}: utterance {u} differs from it alone"
