"""Prompted generation (nvwn_prime_from_score): the scorer runs a prompt's teacher-forced steps all at once, the prime moves its layer
fronts into the history ring and its last two codes into the fed-back indices, and generation continues from sample P.  Checked on
every fp16 kernel variant: the ring bits the prime writes (and the ones it must not), the continuation against the oracle, window
invariance, independence from the scoring stream, every error rule, and NVWaveNet.infer(prompt=...)."""
import ctypes as C

import numpy as np
import pytest
import torch

import nv_wavenet_b200 as nw
from nv_wavenet_b200 import _lib
from nv_wavenet_b200.nv_wavenet import column_major
from oracle import pyoracle as po
from tests import refgen
from tests.common import bits_equal
from tests.test_gpu_parity import FP16_KERNELS, _check_sampled_index, _logit_check, _select_fp16_kernel
from tests.test_gpu_zz_score_stream import _small_net

pytestmark = pytest.mark.gpu

EINVAL, EUNSUPPORTED = -1, -2
KINDS = {"lat": nw.KERNEL_LATENCY, "tc": nw.KERNEL_TENSORCORE, "stream": nw.KERNEL_STREAM}


def _dils(L, md):
    out, d = [], 1
    for _ in range(L):
        out.append(d)
        d *= 2
        if d > md:
            d = 1
    return out


def _engine(w, L, md, B, N, R=64, S=256, A=256, impl=nw.AUTO):
    e = nw.NVWavenetInfer(L, md, B, N, impl, True, R=R, S=S, A=A, dtype=nw.FP16)
    e.load(w)
    return e


def _history(e, batch):
    """The whole ring as fp32 [(maxDil+1)][L][batch][R], read at the stride of a run of `batch` utterances."""
    lib = _lib.lib()
    lib.nvwn_debug_get_history.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    out = np.empty((e.max_dilation + 1, e.L, batch, e.R), np.float32)
    assert lib.nvwn_debug_get_history(e._h, C.c_void_p(out.ctypes.data), batch) == 0
    return out


def _primed_entries(e, P, Bs):
    """{(layer, t): values [Bs][R]} of the ring entries a prime at P writes: layer l at times [max(0, P - d_l), P)."""
    h = _history(e, Bs)
    return {(l, t): h[t % (e.max_dilation + 1), l] for l, d in enumerate(_dils(e.L, e.max_dilation)) for t in range(max(0, P - d), P)}


def _prompted(e, lh, audio, P, Bs):
    """Conditioning of [0, N), the prompt audio[:Bs, :P] scored from 0, then the prime."""
    e.set_conditioning(lh, 0, e.N)
    e.score_stream(audio[:Bs, :P], 0, batch_size=Bs)
    e.prime_from_score()


def test_history_exactly(monkeypatch):
    """The entries a prime writes are bit-identical on all seven variants and within the fp16 tolerance of the ring forced generation
    of the prompt leaves; every other byte of the ring (rows >= Bs included) keeps its bits.  P = 1, 2, < maxDil, > maxDil + 1."""
    L, md, B, N = 12, 16, 20, 64
    w = refgen.lively_inputs(71, 64, 256, 256, L, B, N)
    audio = np.random.default_rng(71).integers(0, 256, (B, N)).astype(np.int32)
    for P in (1, 2, 9, 40):
        seen = {}                                                        # (layer, t) -> the widest rows any variant wrote
        for kernel in FP16_KERNELS:
            _select_fp16_kernel(kernel, monkeypatch)
            Bs = B if kernel.startswith("tc") else 13                    # the whole-batch tensor-core path primes all B rows
            e = _engine(w, L, md, B, N)
            e.set_inputs(w["Lh"], w["selectors"])
            e.run_stream(0, 30, B)                                       # every entry holds something before the prime
            before = _history(e, B).reshape(-1)
            _prompted(e, w["Lh"], audio, P, Bs)
            after = _history(e, B).reshape(-1)
            got = _primed_entries(e, P, Bs)
            # where entry (slot, layer, b < Bs) of a run of Bs utterances sits in the B-stride readback of the whole ring: the plain
            # ring is read at the run's stride, the tiled ones at the engine's
            if kernel == "stream":
                idx = np.arange((md + 1) * L * Bs * 64).reshape(md + 1, L, Bs, 64)
            else:
                idx = np.arange(before.size).reshape(md + 1, L, B, 64)[:, :, :Bs]
            written = np.zeros(before.size, bool)
            for (l, t) in got:
                written[idx[t % (md + 1), l].reshape(-1)] = True
            assert bits_equal(before[~written], after[~written]), f"{kernel}, P = {P}: the prime changed other entries"
            for key, v in got.items():
                if key in seen:
                    rows = min(Bs, seen[key].shape[0])
                    assert bits_equal(seen[key][:rows], v[:rows]), f"{kernel}, P = {P}: entry {key} differs between variants"
                if key not in seen or seen[key].shape[0] < Bs:
                    seen[key] = v
            e.close()
        # forced generation of the same prompt on the whole batch
        _select_fp16_kernel("lat", monkeypatch)
        f = _engine(w, L, md, B, N)
        f.set_inputs(w["Lh"], w["selectors"])
        f.set_forced(audio)
        f.run_stream(0, P, B)
        hist = _history(f, B)
        for (l, t), v in seen.items():
            ref = hist[t % (md + 1), l, :v.shape[0]]
            scale = np.abs(hist[:, l]).max()
            assert np.abs(v - ref).max() <= 2e-2 * scale, f"P = {P}: layer {l}, t = {t} off by {np.abs(v - ref).max() / scale} of its scale"


def _oracle_trace(w, L, md, B, N, forced, R, S, A, prec):
    o = po.Oracle(L, B, N, R, S, A, md, math=po.MATH_PORTABLE, prec=prec)
    o.load(w)
    o.set_inputs(w["Lh"], w["selectors"])
    o.set_forced(forced)
    trace = np.zeros((N, B, A), np.float32)
    o.set_logit_trace(trace)
    o.run(N, B)
    return o, trace


CONTINUATIONS = [(64, 256, 20, 16, 8, 40, kernel) for kernel in FP16_KERNELS] + [
    (32, 128, 6, 8, 4, 21, "stream"),
    (128, 256, 30, 32, 4, 50, "stream"),
    (64, 256, 4, 512, 4, 777, "lat_single"),
    (64, 256, 4, 512, 4, 300, "stream"),
]


@pytest.mark.parametrize("shape", CONTINUATIONS, ids=[f"R{c[0]}_S{c[1]}_L{c[2]}_md{c[3]}_P{c[5]}_{c[6]}" for c in CONTINUATIONS])
def test_continuation_against_the_oracle(shape, monkeypatch):
    """Prime at P, then a teacher-forced continuation of G = maxDil steps (every front entry of the largest dilation is read), one
    launch per step with dumps: each step's logits within the fp16 rule of the fp16-contract and fp32 oracles forced over [0, P + G),
    and the last step's xt / skip within 2e-2."""
    R, S, L, md, B, P, kernel = shape
    A, G = 256, md
    N = P + G
    _select_fp16_kernel(kernel, monkeypatch)
    w = refgen.lively_inputs(72 + P, R, S, A, L, B, N)
    forced = np.random.default_rng(P).integers(0, A, (B, N)).astype(np.int32)
    e = _engine(w, L, md, B, N, R, S, A)
    _prompted(e, w["Lh"], forced, P, B)
    e.set_selectors(w["selectors"])
    e.set_forced(forced)
    za = np.empty((G, B, A), np.float32)
    for g in range(G):
        e.run_stream(P + g, 1, B, dump_activations=True)
        za[g] = e.get_za()
    assert e.launch_info()["kernel"] == {"stream": 16, "lat": 18, "lat_single": 18}.get(kernel, 17)
    o16, t16 = _oracle_trace(w, L, md, B, N, forced, R, S, A, po.PREC_FP16)
    o32, t32 = _oracle_trace(w, L, md, B, N, forced, R, S, A, po.PREC_FP32)
    for g in range(G):
        _logit_check(t16[P + g], za[g], 1e-2)
        _logit_check(t32[P + g], za[g], 1e-2)
    ag, ao = e.activations(), o16.activations()
    for k in ("xt", "skip"):
        sc = np.abs(ao[k]).max()
        assert np.abs(ag[k] - ao[k]).max() <= 2e-2 * sc, f"{k}: {np.abs(ag[k] - ao[k]).max() / sc}"


@pytest.mark.parametrize("kernel", FP16_KERNELS)
def test_free_running_first_sample(kernel, monkeypatch):
    """Without forcing, the index sampled at step P is the first class whose cumulative dumped p exceeds its selector."""
    L, md, B, N, P = 12, 16, 8, 64, 23
    _select_fp16_kernel(kernel, monkeypatch)
    w = refgen.lively_inputs(73, 64, 256, 256, L, B, N)
    audio = np.random.default_rng(73).integers(0, 256, (B, N)).astype(np.int32)
    e = _engine(w, L, md, B, N)
    _prompted(e, w["Lh"], audio, P, B)
    e.set_selectors(w["selectors"])
    e.run_stream(P, 1, B, dump_activations=True)
    y = np.zeros((B, 1), np.int32)
    e.get_yout_stream(y, P, 1)
    _check_sampled_index(e.get_p(), w["selectors"][P], y[:, 0])


def _calls(first, total, W):
    """Uneven calls of at most W samples over [first, first + total)."""
    sizes = [W, max(1, W - 2), 1, (W + 1) // 2, 2]
    out, i = [], 0
    while total > 0:
        n = min(sizes[i % len(sizes)], total)
        out.append((first, n))
        first += n; total -= n; i += 1
    return out


def _continue_windowed(e, lh, audio, P, G, seed, W, B):
    """Prompt scored in uneven calls of <= W samples, the prime, then generation of [P, P + G) in uneven calls: (yOut, last dumps)."""
    for first, n in _calls(0, P, W):
        e.set_conditioning_stream(lh[first:first + n], first)
        e.score_stream(audio[:, first:first + n], first)
    e.prime_from_score()
    y = np.zeros((B, P + G), np.int32)
    calls = _calls(P, G, W)
    for k, (first, n) in enumerate(calls):
        e.set_conditioning_stream(lh[first:first + n], first)
        e.set_selectors_random_stream(seed, first, n)
        e.run_stream(first, n, B, dump_activations=k == len(calls) - 1)
        e.get_yout_stream(y[:, first:first + n], first, n)
    e.synchronize()
    return y[:, P:], e.activations()


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_window_invariance(kind):
    """Scoring and generation through engines of W in {7, 64, 100} samples, P not a multiple of W, uneven calls across the wrap: the
    sampled indices and the last step's dumps equal one engine of the whole length, bit for bit."""
    L, md, B, P, G, seed = 14, 64, 8, 150, 120, 0xA11CE
    w = refgen.lively_inputs(74, 64, 256, 256, L, B, P + G)
    lh = w["Lh"]
    audio = np.random.default_rng(74).integers(0, 256, (B, P)).astype(np.int32)
    ref = _continue_windowed(_engine(w, L, md, B, P + G, impl=KINDS[kind]), lh, audio, P, G, seed, P + G, B)
    assert len(np.unique(ref[0])) > 16
    for W in (7, 64, 100):
        got = _continue_windowed(_engine(w, L, md, B, W, impl=KINDS[kind]), lh, audio, P, G, seed, W, B)
        assert np.array_equal(ref[0], got[0]), f"W = {W}: samples differ"
        for k in ref[1]:
            assert bits_equal(ref[1][k], got[1][k]), f"W = {W}: the {k} dump differs"


def _generate(e, lh, first, n, B, seed=5):
    e.set_conditioning_stream(lh[first:first + n], first)
    e.set_selectors_random_stream(seed, first, n)
    e.run_stream(first, n, B)
    y = np.zeros((e.B, n), np.int32)
    e.get_yout_stream(y, first, n)
    e.synchronize()
    return y[:B]


@pytest.mark.parametrize("kind", ["lat", "tc"])
def test_separation(kind):
    """Scoring after a prime and after generation from it equals scoring without either; priming twice equals priming once;
    reset_history after a prime gives a fresh engine's bits."""
    L, md, B, N, P, k = 12, 16, 16, 128, 37, 30
    w = refgen.lively_inputs(75, 64, 256, 256, L, B, N)
    lh = w["Lh"]
    audio = np.random.default_rng(75).integers(0, 256, (B, N)).astype(np.int32)
    whole = _engine(w, L, md, B, N, impl=KINDS[kind])
    whole.set_conditioning(lh, 0, N)
    ref = whole.score(audio[:, :P + k])

    e = _engine(w, L, md, B, N, impl=KINDS[kind])
    _prompted(e, lh, audio, P, B)
    once = _generate(e, lh, P, 20, B)
    assert bits_equal(ref[:, P:P + k], e.score_stream(audio[:, P:P + k], P)), "the scoring stream changed under a prime and generation"

    twice = _engine(w, L, md, B, N, impl=KINDS[kind])
    _prompted(twice, lh, audio, P, B)
    twice.prime_from_score()
    assert np.array_equal(once, _generate(twice, lh, P, 20, B))
    # the prime leaves the stream open and unchanged: continuing it gives the whole-length bits
    assert bits_equal(ref[:, P:P + k], twice.score_stream(audio[:, P:P + k], P))
    assert bits_equal(ref[:, :P], twice.score_stream(audio[:, :P], 0)), "a fresh stream after a prime"

    fresh = _engine(w, L, md, B, N, impl=KINDS[kind])
    fresh.reset_history()
    expect = _generate(fresh, lh, 0, 40, B)
    twice.reset_history()
    assert np.array_equal(expect, _generate(twice, lh, 0, 40, B)), "reset_history after a prime"


def _rc(e, stream=None):
    lib = _lib.lib()
    code = lib.nvwn_prime_from_score(None if e is None else e._h, stream)
    return code, lib.nvwn_last_error().decode()


def test_errors():
    """Every refusal names the call, and leaves the next sample and the following generation bits as they were."""
    L, md, B, N = 12, 16, 16, 64
    w = refgen.lively_inputs(76, 64, 256, 256, L, B, N)
    lh = w["Lh"]
    audio = np.random.default_rng(76).integers(0, 256, (B, N)).astype(np.int32)

    def refused(kind, setup, code, text):
        """after generation of [0, 10) and setup(e), a refused prime: the engine goes on from 10 with the bits of an engine that had
        the same calls but the prime"""
        out = []
        for attempt in (True, False):
            e = _engine(w, L, md, B, N, impl=KINDS[kind])
            e.reset_history()
            _generate(e, lh, 0, 10, B)
            setup(e)
            if attempt:
                got, msg = _rc(e)
                assert got == code and "nvwn_prime_from_score" in msg and text in msg, f"{got}: {msg}"
            out.append(_generate(e, lh, 10, 12, B))
        assert np.array_equal(out[0], out[1]), text

    def scored(bs=B):
        def setup(e):
            e.set_conditioning(lh, 0, N)
            e.score_stream(audio[:bs, :20], 0, batch_size=bs)
        return setup

    code, msg = _rc(None)
    assert code == EINVAL and "nvwn_prime_from_score: NULL engine" in msg
    refused("lat", lambda e: None, EINVAL, "first_sample = 0")                          # never scored
    refused("lat", lambda e: (e.set_conditioning(lh, 0, N), e.score(audio[:, :20])), EINVAL, "first_sample = 0")     # nvwn_score ends it
    refused("lat", lambda e: (scored()(e), e.set_out_weights(w["Wzs"], w["Bzs"], w["Wza"], w["Bza"])), EINVAL,
            "first_sample = 0")                                                         # a weight change ends it
    refused("tc", scored(8), EINVAL, "tensor-core")
    refused("lat", lambda e: (e.restart_slots([3]), scored(8)(e)), EINVAL, "per-slot")
    e32 = nw.NVWavenetInfer(L, md, B, N, R=64, S=256, A=256, dtype=nw.FP32)
    code, msg = _rc(e32)
    assert code == EUNSUPPORTED and "NVWN_FP16" in msg and "nvwn_prime_from_score" in msg
    # after a prime of 8 utterances, runs of another batch_size are refused until reset_history
    e = _engine(w, L, md, B, N)
    e.reset_history()
    scored(8)(e)
    assert _rc(e)[0] == 0
    with pytest.raises(nw.NvwnError, match=r"nvwn_run_stream: after nvwn_prime_from_score runs need batch_size equal to the primed batch_size \(8\)"):
        e.run_stream(20, 4, B)
    e.run_stream(20, 4, 8)
    e.reset_history()
    e.run_stream(0, 4, B)


def test_nvwavenet_infer_prompt():
    """The prompt columns come back as given; window=W equals no window bit for bit; the result equals the engine calls spelled out,
    for seeded and host-drawn selectors, host and CUDA prompts."""
    net, Lm, g = _small_net(77)
    R, A = net.R, net.A
    Bn, Nn, P = 3, 250, 100
    cond = (0.5 * torch.randn(2 * R, Bn, Lm, Nn, generator=g)).cuda()
    prompt = torch.randint(0, A, (Bn, P), generator=g).to(torch.int32)
    libc = C.CDLL(None)
    for seed in (1234, None):
        def run(**kw):
            if seed is None:
                libc.srand(99)
            return net.infer(cond, 0, seed=seed, fp16=True, prompt=kw.pop("prompt", prompt), **kw).cpu().numpy()
        whole = run()
        assert np.array_equal(whole[:, :P], prompt.numpy())
        for W in (7, 64, 100):
            assert np.array_equal(whole, run(window=W)), f"seed {seed}, W = {W}"
        assert np.array_equal(whole, run(prompt=prompt.cuda().to(torch.int64)))
        # spelled out on the engine infer() used
        eng = net._engine(Bn, Nn, True)
        eng.reset_history()
        eng.set_conditioning(column_major(cond).float(), 0, Nn)
        eng.score_stream(prompt.numpy(), 0)
        eng.prime_from_score()
        if seed is None:
            libc.srand(99)
            sel = np.empty(Nn * Bn, np.float32)
            assert _lib.lib().nvwn_libc_selectors(C.c_void_p(sel.ctypes.data), Bn, Nn) == 0
            eng.set_selectors(sel)
        else:
            eng.set_selectors_random(seed)
        eng.run_stream(P, Nn - P, Bn)
        y = np.zeros((Bn, Nn), np.int32)
        eng.get_yout(y, 0, Nn)
        eng.synchronize()
        assert np.array_equal(whole[:, P:], y[:, P:]), f"seed {seed}: infer(prompt=...) differs from the engine calls"


def test_c3_first_step_logits():
    """C3 (L20 R64 S256, maxDil 512), 64 utterances of 20 000 samples, P = 16 000: the first continuation step's logits after a prime
    are within the fp16 rule of a forced-generation engine's at the same step."""
    L, md, B, N, P = 20, 512, 64, 20000, 16000
    w = refgen.lively_inputs(78, 64, 256, 256, L, 1, 1)
    gen = torch.Generator(device="cuda").manual_seed(78)
    lh = 0.5 * torch.randn((1000, L, B, 128), generator=gen, device="cuda")           # repeated every 1 000 samples
    audio = torch.randint(0, 256, (B, N), generator=gen, device="cuda", dtype=torch.int32)
    za = {}
    for arm in ("forced", "primed"):
        e = _engine(w, L, md, B, N)
        for k in range(N // 1000):
            e.set_conditioning(lh, 1000 * k, 1000)
        e.set_selectors_random(1)
        e.reset_history()
        if arm == "forced":
            e.set_forced(audio)
            e.run_stream(0, P + 1, B, dump_activations=True)
        else:
            e.score_stream(audio[:, :P], 0)
            e.prime_from_score()
            e.set_forced(audio)
            e.run_stream(P, 1, B, dump_activations=True)
        e.synchronize()
        za[arm] = e.get_za()
        e.close()
        del e
        torch.cuda.empty_cache()
    assert np.isfinite(za["primed"]).all()
    _logit_check(za["forced"], za["primed"], 1e-2)
