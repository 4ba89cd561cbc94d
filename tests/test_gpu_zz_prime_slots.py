"""Prompted continuous batching (nvwn_prime_slots_from_score, NVWaveNet.infer_many(prompts=...)): single slots of a running engine are
primed from rows of a scoring stream.  Checked on every fp16 kernel variant: the ring bits a slot prime writes and the ones it must not,
at early, late and wrapped engine times; continuations served through a queue against infer(prompt=...) of each utterance alone; the
rows that were not primed before and after an early prime; the scoring stream's independence; the primed slots' selectors; every
error rule."""
import ctypes as C

import numpy as np
import pytest
import torch

import nv_wavenet_b200 as nw
from nv_wavenet_b200 import _lib
from nv_wavenet_b200.nv_wavenet import Impl
from tests import refgen
from tests.common import bits_equal
from tests.test_gpu_parity import FP16_KERNELS, _select_fp16_kernel
from tests.test_gpu_zz_prime import _dils, _engine, _history
from tests.test_gpu_zz_score_stream import _small_net
from tests.test_gpu_zz_selectors import _net, philox_selectors

pytestmark = pytest.mark.gpu

EINVAL, EUNSUPPORTED = -1, -2
L, MD, B, N, BS = 12, 16, 20, 64, 5          # engines of 20 slots and 64 samples; scoring streams of 5 rows
ROWS, SLOTS, SEEDS = [3, 0, 4], [B - 1, 7, 2], [11, 12, 13]


def _pieces(first, end, W):
    """[first, end) in pieces of at most W samples that do not cross a multiple of W."""
    out = []
    while first < end:
        m = min(end - first, W - first % W)
        out.append((first, m))
        first += m
    return out


def _score_rows(e, lh, audio, P):
    """Scores audio[:k, :P] on e through its store rows 0..k-1 (set_conditioning_slots), lh [P][L][k][2R], windows of e.N."""
    k = audio.shape[0]
    for a, m in _pieces(0, P, e.N):
        e.set_conditioning_slots(np.ascontiguousarray(lh[a:a + m]), list(range(k)), a)
        e.score_stream(audio[:, a:a + m], a)


def _generate(e, lh, first, n, seed=5, dump=False):
    """Samples [first, first + n) of every slot, conditioning lh [T][L][B][2R] at those samples and selectors under `seed`."""
    y = np.zeros((e.B, n), np.int32)
    for a, m in _pieces(first, first + n, e.N):
        e.set_conditioning_stream(lh[a:a + m], a)
        e.set_selectors_random_stream(seed, a, m)
        e.run_stream(a, m, e.B, dump_activations=dump and a + m == first + n)
        e.get_yout_stream(y[:, a - first:a - first + m], a, m)
    e.synchronize()
    return y


def _inputs(seed, T):
    w = refgen.lively_inputs(seed, 64, 256, 256, L, B, T)
    audio = np.random.default_rng(seed).integers(0, 256, (BS, T)).astype(np.int32)
    lhs = np.ascontiguousarray(w["Lh"][:, :, :BS])                          # the prompts' conditioning, [T][L][BS][2R]
    return w, audio, lhs


_REF = {}


def _one_utterance_ring(w, lhs, audio, r, P):
    """The ring of nvwn_prime_from_score of prompt row r alone on a one-utterance engine: [(MD+1)][L][R]."""
    key = (r, P)
    if key not in _REF:
        f = _engine(w, L, MD, 1, N, impl=nw.KERNEL_LATENCY)
        f.reset_history()
        for a, m in _pieces(0, P, N):
            f.set_conditioning_stream(np.ascontiguousarray(lhs[a:a + m, :, r:r + 1]), a)
            f.score_stream(audio[r:r + 1, a:a + m], a)
        f.prime_from_score()
        _REF[key] = _history(f, 1)[:, :, 0]
        f.close()
    return _REF[key]


@pytest.mark.parametrize("kernel", FP16_KERNELS)
def test_ring_bits(kernel, monkeypatch):
    """Slot primes at t0 in {0, 5 (< maxDil), 40, 90 (the 64-sample store wrapped)}, P in {1, 9 (< d_max = 16), 100 (> N)}: each primed
    slot's ring row equals the one-utterance prime of its prompt, shifted by t0 - P, bit for bit, and is zero elsewhere; every other
    row keeps its bits but for the entries of the negative times, which the first prime before maxDil zeroes in every row."""
    _select_fp16_kernel(kernel, monkeypatch)
    w, audio, lhs = _inputs(81, 100)
    M = MD + 1
    dils = _dils(L, MD)
    for t0 in (0, 5, 40, 90):
        for P in (1, 9, 100):
            e = _engine(w, L, MD, B, N)
            e.reset_history()
            _generate(e, w["Lh"], 0, 30)                                 # every entry holds something ...
            e.reset_history()                                            # ... which the reset leaves there
            if t0:
                _generate(e, w["Lh"], 0, t0)
            _score_rows(e, lhs, audio, P)
            before = _history(e, B)
            e.prime_slots_from_score(ROWS, SLOTS, SEEDS)
            after = _history(e, B)
            others = [b for b in range(B) if b not in SLOTS]
            want = before[:, :, others].copy()
            if t0 < MD:
                want[t0:M] = 0                                           # times [t0 - M, 0)
            assert bits_equal(want, after[:, :, others]), f"{kernel}, t0 = {t0}, P = {P}: other rows changed"
            for r, s in zip(ROWS, SLOTS):
                ref = _one_utterance_ring(w, lhs, audio, r, P)
                exp = np.zeros((M, L, e.R), np.float32)
                for l, d in enumerate(dils):
                    for tau in range(max(0, P - d), P):
                        exp[(t0 - P + tau) % M, l] = ref[tau % M, l]
                assert bits_equal(exp, after[:, :, s]), f"{kernel}, t0 = {t0}, P = {P}: slot {s} (row {r})"
            e.close()


def _queue(seed, lengths, plens, Lm, R):
    g = torch.Generator().manual_seed(seed)
    conds = [(0.5 * torch.randn(2 * R, Lm, n, generator=g)).cuda() for n in lengths]
    prompts = [None if p is None else torch.randint(0, 256, (p,), generator=g).to(torch.int32) for p in plens]
    seeds = [1000 + 7 * u for u in range(len(lengths))]
    return conds, prompts, seeds


def _check_queue(net, conds, prompts, seeds, slots, window):
    timing = {}
    got = net.infer_many(conds, seeds, slots=slots, window=window, fp16=True, timing=timing, prompts=prompts)
    assert set(timing) == {"restart_upload_s", "generate_s", "prime_s"} and timing["prime_s"] > 0
    plain = net.infer_many(conds, seeds, slots=slots, window=window, fp16=True)
    for u, c in enumerate(conds):
        p = prompts[u]
        kw = {} if p is None else dict(prompt=p[None])
        want = net.infer(c[:, None].contiguous(), Impl.AUTO, seed=seeds[u], fp16=True, **kw)[0].cpu().numpy()
        y = got[u].cpu().numpy()
        assert y.shape == (c.size(2),)
        assert np.array_equal(want, y), f"utterance {u} (prompt {None if p is None else p.numel()}) differs from infer() alone"
        if p is None:
            assert np.array_equal(plain[u].cpu().numpy(), y), f"utterance {u}: infer_many without prompts differs"
        else:
            assert np.array_equal(y[:p.numel()], p.numpy())
    return got


@pytest.mark.parametrize("kernel", FP16_KERNELS)
def test_infer_many_prompts(kernel, monkeypatch):
    """A queue through 4 slots and windows of 50: prompted and unprompted utterances, two prompt lengths at boundary 0 (30 and 70, longer
    than the window), prompted starts at later boundaries, two prompts of one length at one boundary.  Every output equals infer() of
    that utterance alone with its prompt, and the unprompted ones equal infer_many without prompts."""
    _select_fp16_kernel(kernel, monkeypatch)
    net, Lm, _ = _small_net(82)
    lengths = [120, 90, 200, 75, 130, 60, 110, 140, 95]
    plens = [None, 30, 70, None, 30, 12, None, 45, 45]
    conds, prompts, seeds = _queue(82, lengths, plens, Lm, net.R)
    got = _check_queue(net, conds, prompts, seeds, 4, 50)
    assert len(np.unique(got[2].cpu().numpy()[70:])) > 16


def test_infer_many_prompts_c3():
    """C3 (L20 R64 S256, maxDil 512), 16 slots, windows of 4 000: 24 utterances of 6 000-14 000 samples, most prompted with 1-9 000
    samples (several longer than a window)."""
    Lm, md = 20, 512
    w = refgen.lively_inputs(83, 64, 256, 256, Lm, 1, 1)
    net = _net(w, Lm, 64, 256, 256, md)
    rng = np.random.default_rng(83)
    lengths = [int(v) for v in rng.integers(6000, 14000, 24)]
    plens = [None if u % 4 == 3 else int(rng.integers(1, min(9000, n - 1))) for u, n in enumerate(lengths)]
    plens[0] = 1
    conds, prompts, seeds = _queue(83, lengths, plens, Lm, 64)
    _check_queue(net, conds, prompts, seeds, 16, 4000)


@pytest.mark.parametrize("kernel", FP16_KERNELS)
def test_early_prime_leaves_other_rows(kernel, monkeypatch):
    """Rows that were not primed give the same samples and last-step dumps whether or not slot 0 was primed at t0 = 5 < maxDil (after
    which every launch reads the ring at every step)."""
    _select_fp16_kernel(kernel, monkeypatch)
    w, audio, lhs = _inputs(84, 100)
    t0, P, G = 5, 23, 60
    out = {}
    for primed in (False, True):
        e = _engine(w, L, MD, B, N)
        e.reset_history()
        _generate(e, w["Lh"], 0, 30)
        e.reset_history()
        _generate(e, w["Lh"], 0, t0)
        if primed:
            _score_rows(e, lhs[:, :, :1], audio[:1], P)
            e.prime_slots_from_score([0], [0], [9])
        else:
            e.set_conditioning_slots(np.ascontiguousarray(lhs[:1, :, :1]), [0], 0)    # a per-slot call in both arms
        y = _generate(e, w["Lh"], t0, G, dump=True)
        out[primed] = (y, e.activations())
        e.close()
    rest = list(range(1, B))
    assert np.array_equal(out[False][0][rest], out[True][0][rest]), f"{kernel}: samples of rows that were not primed"
    assert len(np.unique(out[True][0][rest])) > 16
    for k, v in out[False][1].items():
        ax = 1 if k in ("xt", "skip") else 0
        assert bits_equal(np.take(v, rest, axis=ax), np.take(out[True][1][k], rest, axis=ax)), f"{kernel}: the {k} dump"


@pytest.mark.parametrize("kernel", FP16_KERNELS)
def test_scoring_stream_independent(kernel, monkeypatch):
    """After a slot prime, and after generation from it, the scoring stream goes on with the bits of a stream that was never primed."""
    _select_fp16_kernel(kernel, monkeypatch)
    w, audio, lhs = _inputs(85, 100)
    P, k = 40, 30
    ref = _engine(w, L, MD, B, N)
    ref.reset_history()
    _score_rows(ref, lhs, audio, P)
    ref.set_conditioning_slots(np.ascontiguousarray(lhs[P:P + k]), list(range(BS)), P)
    want = ref.score_stream(audio[:, P:P + k], P)
    e = _engine(w, L, MD, B, N)
    e.reset_history()
    _generate(e, w["Lh"], 0, 10)
    _score_rows(e, lhs, audio, P)
    e.prime_slots_from_score(ROWS, SLOTS, SEEDS)
    e.prime_slots_from_score([1], [5])                                   # a later prime from the same stream
    e.set_conditioning_slots(np.ascontiguousarray(lhs[P:P + k]), list(range(BS)), P)
    # generation reads and writes nothing of the stream: slots 0..4 hold the scoring conditioning, the others their own
    e.set_selectors_random_slots(10, 20)
    e.run_stream(10, 20, B)
    e.synchronize()
    assert bits_equal(want, e.score_stream(audio[:, P:P + k], P)), f"{kernel}: the scoring stream changed"


def test_selectors_of_a_primed_slot():
    """set_selectors_random_slots of a slot primed at t0 with a prompt of P samples draws counter tau = t - (t0 - P) under its seed:
    the samples equal those of host selectors restated with Philox, on every row."""
    w, audio, lhs = _inputs(86, 100)
    t0, P, G, seed = 30, 45, 50, 0xBEEF
    ys = []
    for host in (False, True):
        e = _engine(w, L, MD, B, N)
        e.reset_history()
        _generate(e, w["Lh"], 0, t0)
        _score_rows(e, lhs[:, :, :2], audio[:2], P)
        e.prime_slots_from_score([1], [6], [seed])
        e.set_conditioning_stream(w["Lh"][t0:t0 + G], t0)
        if host:
            sel = np.zeros((N, B), np.float32)
            rest, mine = philox_selectors(t0 + G, 0)[t0:], philox_selectors(P + G, seed)[P:]     # the reset left origin 0, key 0
            for i in range(G):
                sel[(t0 + i) % N] = rest[i]
                sel[(t0 + i) % N, 6] = mine[i]
            e.set_selectors(sel)
        else:
            e.set_selectors_random_slots(t0, G)
        e.run_stream(t0, G, B)
        y = np.zeros((B, G), np.int32)
        e.get_yout_stream(y, t0, G)
        e.synchronize()
        ys.append(y)
        e.close()
    assert np.array_equal(ys[0], ys[1])
    assert len(np.unique(ys[0][6])) > 8


def _rc(e, rows, slots, n=None, seeds=None):
    lib = _lib.lib()
    arr = lambda v, t: None if v is None else np.ascontiguousarray(v, dtype=t)
    r, s, k = arr(rows, np.int32), arr(slots, np.int32), arr(seeds, np.uint64)
    ptr = lambda a: None if a is None else C.c_void_p(a.ctypes.data)
    n = (0 if s is None else s.size) if n is None else n
    code = lib.nvwn_prime_slots_from_score(None if e is None else e._h, ptr(r), ptr(s), n, ptr(k), None)
    return code, lib.nvwn_last_error().decode()


def test_errors():
    """Every refusal returns the stated code with a message that names the call, and leaves the ring, the fed-back indices (the
    following generation) and the scoring stream as they were."""
    w, audio, lhs = _inputs(87, 100)
    P = 20

    def setup(e, scored=True):
        e.reset_history()
        _generate(e, w["Lh"], 0, 10)
        if scored:
            _score_rows(e, lhs[:, :, :4], audio[:4], P)
        else:
            e.set_conditioning_slots(np.ascontiguousarray(lhs[:1, :, :1]), [0], 0)

    def after(e, scored=True):
        h = _history(e, B)
        lp = None
        if scored:
            e.set_conditioning_slots(np.ascontiguousarray(lhs[P:P + 10, :, :4]), list(range(4)), P)
            lp = e.score_stream(audio[:4, P:P + 10], P)
        return h, lp, _generate(e, w["Lh"], 10, 12)

    want = {}
    for scored in (True, False):
        e = _engine(w, L, MD, B, N)
        setup(e, scored)
        want[scored] = after(e, scored)
        e.close()

    def refused(rows, slots, text, n=None, scored=True, code=EINVAL):
        e = _engine(w, L, MD, B, N)
        setup(e, scored)
        h0 = _history(e, B)
        got, msg = _rc(e, rows, slots, n)
        assert got == code and "nvwn_prime_slots_from_score" in msg and text in msg, f"{got}: {msg}"
        assert bits_equal(h0, _history(e, B)), text
        h, lp, y = after(e, scored)
        assert bits_equal(want[scored][0], h) and np.array_equal(want[scored][2], y), text
        if scored:
            assert bits_equal(want[scored][1], lp), text
        e.close()

    code, msg = _rc(None, [0], [0])
    assert code == EINVAL and "nvwn_prime_slots_from_score: NULL engine" in msg
    refused([0], [0], "no open scoring stream", scored=False)
    refused(None, [0], "rows is NULL")
    refused([0], None, "slots is NULL", n=1)
    refused([4], [0], "row 4 is outside [0, 4)")
    refused([-1], [0], "row -1 is outside")
    refused([1, 1], [0, 2], "row 1 is given twice")
    refused([0], [B], f"slot {B} is outside")
    refused([0, 1], [3, 3], "slot 3 is given twice")
    refused([0], [0], "need 1 <= n", n=0)
    e32 = nw.NVWavenetInfer(L, MD, B, N, R=64, S=256, A=256, dtype=nw.FP32)
    code, msg = _rc(e32, [0], [0])
    assert code == EUNSUPPORTED and "NVWN_FP16" in msg and "nvwn_prime_slots_from_score" in msg
