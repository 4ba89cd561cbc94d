"""The last stage of every generation kernel: softmax of the logits, then the first class whose cumulative probability exceeds
the selector.  Each kernel writes that stage its own way (one thread, a warp per utterance, 8 classes per lane with a shuffle
scan, four 64-class parts per utterance), so each one is checked here where such scans go wrong.

A. Exactly known distributions.  With the output layer's weights at zero every kernel's logits are its output bias: `base` on a
   support set of m classes and `base - 160` elsewhere, all exact in fp16.  With `base` 0 or a power of two, every exp of the
   fp16 / FP32_FAST kernels is exactly 1 on the support and 0 off it, so the running sums are exact integers, the total is m, the
   target is fl32(sel * m) and the sampled index is support[floor(target)]: checked at every step, with no tolerance.  The
   bit-exact fp32 kernel must equal the CPU model bit for bit, and the scorer's logp must be -log m and -160 - log m.

B. Shifted logits.  Softmax does not change when a constant is added to every logit, and training does not pin that constant:
   lively logits shifted by up to -100 must give the same distribution, finite, within each kernel's tolerance.
"""
import numpy as np
import pytest

import nv_wavenet_b200 as nw
from nv_wavenet_b200 import _lib
from tests import refgen
from tests.test_gpu_parity import FP16_KERNELS, _check_sampled_index, _select_fp16_kernel, assert_acts_bit_equal, cpu_oracle, gpu_engine

pytestmark = pytest.mark.gpu

L, B, R, S, MD = 12, 20, 64, 256, 8        # L = 12: the cluster kernel takes the stack; B = 20: ragged 8- and 16-row tiles
OFF = 160.0                                # logits off the support sit this far below it: exp underflows to exactly 0
BASES = [0.0, 64.0, -128.0]
NONEXACT = FP16_KERNELS + ["fp32_fast"]       # every kernel whose softmax runs on ex2.approx
LAUNCHED = {"fp32_fast": 16, "stream": 16, "lat": 18, "lat_single": 18}     # the tensor-core variants: 17


def _engine(kernel, w, B, N, A, monkeypatch):
    """An engine on one of NONEXACT: an fp16 kernel of FP16_KERNELS, or FP32_FAST."""
    if kernel == "fp32_fast":
        return gpu_engine(w, L, B, N, R, S, A, MD, dtype=nw.FP32_FAST)
    _select_fp16_kernel(kernel, monkeypatch)
    return gpu_engine(w, L, B, N, R, S, A, MD, dtype=nw.FP16)


def _assert_launched(e, kernel, batch_per_cta=None):
    info = e.launch_info()
    assert info["kernel"] == LAUNCHED.get(kernel, 17), info
    if kernel.startswith("lat"):
        assert info["cluster"] == (3 if kernel == "lat" else 1), info
    if batch_per_cta is not None:
        assert info["batch_per_cta"] == batch_per_cta, info


def _zero_output_layer(w):
    w = dict(w)
    w["Wza"] = np.zeros_like(w["Wza"])
    return w


def _supports(A):
    """Support sets that put the boundaries of every scan layout inside or at the edge of a support."""
    per = A // 32                                      # classes per lane of the warp-per-utterance scans
    s = {"all": np.arange(A)}
    for c in sorted({0, 7, 8, per - 1, per, 63, 64, A - 1}):
        s[f"onehot{c}"] = np.array([c])
    s["block40"] = np.arange(100, 140)                 # not a power of two; crosses lane boundaries and the 128-class split
    s["lane_last"] = np.arange(per - 1, A, per)        # the last class of every lane
    s["head200"] = np.arange(200)                      # a zero tail: falling back to A - 1 would be wrong
    s["from64"] = np.arange(64, A)                     # the first 64-class part of the tensor-core kernel is empty
    s["random97"] = np.sort(np.random.default_rng(97).choice(A, 97, replace=False))
    return s


def _bza(A, support, base):
    z = np.full(A, base - OFF, np.float32)
    z[support] = base
    return z


def _selectors(m, N, B, seed):
    """[N][B] selectors: 0, every boundary k/m and k/m - 2^-16, 1 - 2^-24 (the largest the device Philox draw gives), and seeded
    multiples of 2^-24, in a seeded order so that the edge cases land on every row of every tile."""
    k = np.arange(1, m, dtype=np.float64)
    edges = np.concatenate([[0.0, 1.0 - 2.0 ** -24], k / m, k / m - 2.0 ** -16]).astype(np.float32)
    assert edges.size <= N * B, "too few (step, utterance) slots for every boundary selector"
    rng = np.random.default_rng(seed)
    rand = (rng.integers(0, 1 << 24, N * B - edges.size) * 2.0 ** -24).astype(np.float32)
    return np.ascontiguousarray(rng.permutation(np.concatenate([edges, rand])).reshape(N, B))


def _expected_indices(sel, support):
    """[B][N] indices a kernel whose exps are exactly 1 on the support and 0 off it must sample: the running sums are exact integers
    and the total is m, so the target fl32(sel * m) falls in the support's floor(target)-th class."""
    m = np.float32(len(support))
    target = sel * m                                   # float32 * float32: the kernel's one multiply, rounded to nearest
    assert target.dtype == np.float32 and (target < m).all()
    return support[np.floor(target).astype(np.int64)].T


def _run(e, w, bza, sel, B, N):
    e.set_out_weights(w["Wzs"], w["Bzs"], w["Wza"], bza)
    e.set_selectors(sel)
    e.reset_history()
    y = np.zeros((B, N), np.int32)
    e.run(N, B, y, dump_activations=True)
    e.synchronize()
    return y, e.get_za(), e.get_p()


def _check_known_distribution(e, w, A, B, N, base, seed):
    for name, sup in _supports(A).items():
        m = len(sup)
        bza = _bza(A, sup, base)
        sel = _selectors(m, N, B, seed + m)
        y, za, p = _run(e, w, bza, sel, B, N)
        what = f"support {name}, base {base}"
        assert np.array_equal(za, np.broadcast_to(bza, za.shape)), f"{what}: the logits are not the output bias"
        want = _expected_indices(sel, sup)
        bad = np.argwhere(y != want)
        if bad.size:
            b, t = bad[0]
            raise AssertionError(f"{what}: {len(bad)} of {y.size} indices wrong; first: utterance {b}, step {t}, selector "
                                 f"{float(sel[t, b])!r}, sampled {y[b, t]}, expected {want[b, t]}")
        on = np.zeros(A, bool)
        on[sup] = True
        pw = np.broadcast_to(np.where(on, np.float32(1) / np.float32(m), np.float32(0)), p.shape)
        bad = np.argwhere(p.view(np.uint32) != pw.view(np.uint32))
        if bad.size:
            b, a = bad[0]
            raise AssertionError(f"{what}: {len(bad)} dumped probabilities differ; first: utterance {b}, class {a}: "
                                 f"{p[b, a]!r}, expected {pw[b, a]!r}")


_CASES = [pytest.param(k, 256, id=k) for k in NONEXACT] + [pytest.param(k, 512, id=f"{k}-A512") for k in ("stream", "fp32_fast")]


@pytest.mark.parametrize("base", BASES)
@pytest.mark.parametrize("kernel, A", _CASES)
def test_known_distributions_sample_exactly(kernel, A, base, monkeypatch):
    """Every step's index and the last step's p of the fp16 and FP32_FAST kernels, exactly.  A = 512: 16 classes per lane."""
    N = 32 if A == 256 else 64                         # room for every boundary selector of the 512-class support
    w = _zero_output_layer(refgen.lively_inputs(61 + A, R, S, A, L, B, N))
    e = _engine(kernel, w, B, N, A, monkeypatch)
    _check_known_distribution(e, w, A, B, N, base, 5)
    _assert_launched(e, kernel, 8 if kernel == "lat" else None)


def test_sixteen_row_cluster_tail_samples_exactly(monkeypatch):
    """400 utterances: more 8-row clusters than stay resident, so the cluster kernel's tail CTA serves two rows per warp."""
    A, Bb, N = 256, 400, 8
    fit8, fit16 = (_lib.lib().nvwn_debug_lat_max_clusters(S, rows) for rows in (8, 16))
    if not (fit8 < (Bb + 7) // 8 and (Bb + 15) // 16 <= fit16):
        pytest.skip(f"{fit8} / {fit16} resident 8- / 16-row clusters: 400 utterances do not fall between the two limits on this device")
    w = _zero_output_layer(refgen.lively_inputs(63, R, S, A, L, Bb, N))
    e = _engine("lat", w, Bb, N, A, monkeypatch)
    for base in BASES:
        _check_known_distribution(e, w, A, Bb, N, base, 7)
        _assert_launched(e, "lat", 16)


@pytest.mark.parametrize("base", [0.0, 64.0, -64.0])    # the CPU model starts the max at 0: exp underflows below about -103
def test_known_distributions_bit_exact_fp32(base):
    """The bit-exact kernel scans sequentially in one thread, as the CPU model does: y, the logits and p equal it bit for bit."""
    A, N = 256, 32
    w = _zero_output_layer(refgen.lively_inputs(65, R, S, A, L, B, N))
    e = gpu_engine(w, L, B, N, R, S, A, MD)
    for name, sup in _supports(A).items():
        bza = _bza(A, sup, base)
        sel = _selectors(len(sup), N, B, 9 + len(sup))
        y, za, p = _run(e, w, bza, sel, B, N)
        o = cpu_oracle(dict(w, Bza=bza, selectors=sel), L, B, N, R, S, A, MD)
        assert np.array_equal(y, o.run(N, B)), f"support {name}, base {base}: indices differ from the CPU model"
        assert np.array_equal(za.view(np.uint32), o.get_za().view(np.uint32)), f"support {name}, base {base}: za"
        assert np.array_equal(p.view(np.uint32), o.get_p().view(np.uint32)), f"support {name}, base {base}: p"


@pytest.mark.parametrize("base", BASES)
def test_known_distributions_scorer(base):
    """logp = -log m on the support and -160 - log m off it, within 4 float32 ulps of the larger of |z| and the logsumexp."""
    A, N = 256, 32
    w = _zero_output_layer(refgen.lively_inputs(67, R, S, A, L, B, N))
    rng = np.random.default_rng(3)
    for impl in (nw.KERNEL_LATENCY, nw.KERNEL_TENSORCORE, nw.KERNEL_STREAM):
        e = gpu_engine(w, L, B, N, R, S, A, MD, dtype=nw.FP16, impl=impl)
        for name, sup in _supports(A).items():
            m = len(sup)
            bza = _bza(A, sup, base)
            e.set_out_weights(w["Wzs"], w["Bzs"], w["Wza"], bza)
            audio = rng.integers(0, A, (B, N)).astype(np.int32)
            audio[:, ::2] = rng.choice(sup, (B, (N + 1) // 2))            # every other sample on the support
            logp = e.score(audio)
            z = bza[audio].astype(np.float64)
            lse = base + np.log(m)
            want = z - lse
            tol = 4 * np.spacing(np.maximum(np.abs(z), abs(lse)).astype(np.float32)).astype(np.float64)
            err = np.abs(logp - want)
            assert np.all(err <= tol), f"impl {impl}, support {name}, base {base}: max error {err.max()} (tolerance {tol.max()})"


# ---------------- B. shifted logits

SHIFTS = [0.0, 96.0, -48.0, -90.0, -100.0]
NS = 24                                                # steps of the shifted-logit runs


def _softmax64(z):
    z = np.asarray(z, np.float64)
    e = np.exp(z - z.max(axis=-1, keepdims=True))      # the true max, not the CPU model's start at 0
    return e / e.sum(axis=-1, keepdims=True)


@pytest.fixture(scope="module")
def shifted():
    """Lively inputs with Bza rounded to multiples of 1/16, so that Bza + c is exact in fp16; the fp32 model's trajectory at c = 0
    as the history of every run; and per shift c, the inputs, the CPU model's teacher-forced indices and activations."""
    A = 256
    w = refgen.lively_inputs(71, R, S, A, L, B, NS)
    w["Bza"] = (np.round(w["Bza"] * 16) / 16).astype(np.float32)
    forced = cpu_oracle(w, L, B, NS, R, S, A, MD).run(NS, B)
    cases = {}
    for c in SHIFTS:
        wc = dict(w, Bza=(w["Bza"] + np.float32(c)).astype(np.float32))
        o = cpu_oracle(wc, L, B, NS, R, S, A, MD)
        o.set_forced(forced)
        y = o.run(NS, B)
        cases[c] = (wc, y, o.activations())
    return forced, cases


def _run_shifted(e, wc):
    e.set_out_weights(wc["Wzs"], wc["Bzs"], wc["Wza"], wc["Bza"])
    e.reset_history()
    y = np.zeros((B, NS), np.int32)
    e.run(NS, B, y, dump_activations=True)
    e.synchronize()
    return y


@pytest.mark.parametrize("kernel", NONEXACT)
def test_shifted_logits(kernel, shifted, monkeypatch):
    """p of the last step: finite, near a float64 softmax of the CPU model's logits, and the same at every shift."""
    A = 256
    forced, cases = shifted
    e = _engine(kernel, cases[0.0][0], B, NS, A, monkeypatch)
    e.set_forced(forced)
    tol = 1e-3 if kernel == "fp32_fast" else 1e-2
    p0 = None
    for c in SHIFTS:
        wc, _, ao = cases[c]
        y = _run_shifted(e, wc)
        _assert_launched(e, kernel)
        p = e.get_p()
        assert np.isfinite(p).all(), f"shift {c}: p not finite"
        ref = _softmax64(ao["za"])
        err = np.abs(p - ref).max() / ref.max()
        assert err <= tol, f"shift {c}: p off the float64 softmax of the CPU model's logits by {err} of its max"
        if p0 is None:
            p0 = p
        else:
            err = np.abs(p - p0).max() / p0.max()
            assert err <= 1e-3, f"shift {c}: p moved by {err} of its max from the unshifted logits"
        _check_sampled_index(p, wc["selectors"][NS - 1], y[:, NS - 1])
        assert ((0 <= y) & (y < A)).all(), f"shift {c}: index out of range"


def test_shifted_logits_bit_exact_fp32(shifted):
    """Down to c = -90 the bit-exact kernel still equals the CPU model, which starts its max at 0."""
    A = 256
    forced, cases = shifted
    e = gpu_engine(cases[0.0][0], L, B, NS, R, S, A, MD)
    e.set_forced(forced)
    for c in (0.0, 96.0, -48.0, -90.0):
        wc, yo, ao = cases[c]
        y = _run_shifted(e, wc)
        assert np.array_equal(y, yo), f"shift {c}: indices differ from the CPU model"
        assert_acts_bit_equal(ao, e.activations())


def test_shifted_logits_scorer(shifted):
    A = 256
    forced, cases = shifted
    e = gpu_engine(cases[0.0][0], L, B, NS, R, S, A, MD, dtype=nw.FP16)
    lp0 = None
    for c in SHIFTS:
        wc = cases[c][0]
        e.set_out_weights(wc["Wzs"], wc["Bzs"], wc["Wza"], wc["Bza"])
        lp = e.score(forced)
        assert np.isfinite(lp).all(), f"shift {c}: logp not finite"
        if lp0 is None:
            lp0 = lp
        else:
            err = np.abs(lp - lp0).max()
            assert err <= 1e-3, f"shift {c}: logp moved by {err} from the unshifted logits"
