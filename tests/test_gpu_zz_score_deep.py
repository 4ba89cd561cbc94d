"""Teacher-forced scoring against the CPU model where a layer's dilation is longer than the scorer's time chunk.

The scorer (wn_score_kernel.cu, driven by score_range in wn_engine.cu) runs a call in chunks of T = min(N, max(1, SCORE_ROWS / B))
steps, sized from the engine's B.  After a chunk of Tc steps every layer moves its last d_l fp16 inputs to the front of its buffer,
in pieces of Tc * Bs rows that do not overlap, and the next chunk reads x_l[t - d_l] from that front.  Where d_l > T a front is
itself made of earlier carries, so a front that keeps the wrong rows shows only where the largest dilation reads across at least two
carries.  A prime (nvwn_prime_from_score) copies the fronts the last chunk left into the history ring, so it inherits any such error.
The other scorer tests compare the scorer with itself (streamed against whole, packed against alone), and both sides of those run
the same carry.  Here the reference is the pinned CPU oracle (MATH_PORTABLE): its fp32 model and its fp16 contract, following
chosen rows only.

Every case has max d_l >= 2 T and N >= max d_l + 2 T (test_score_deep_host.py recomputes that from SCORE_ROWS without a GPU):
- test_scored_against_the_oracle: C3 at the serving batch (B = 64, T = 256, four carries, a ragged last chunk); L10 maxDil 512 at
  B = 2048 (T = 8, so a carry of d = 512 is 64 copies; the conditioning is filled from the device a window at a time); batch_size 150
  on an engine of B = 200 (T = 81, fronts at the stride of 150 rows in buffers laid out for 200); R128 and R32 at B = 128 (T = 128).
  At every step of the followed rows, which score the fp32 oracle's free-running trajectory (the other rows score random codes):
  logits within the fp16 rule of the fp16-contract oracle with mean <= 3e-4 and of the fp32 oracle, logp within 2e-2 max|z| of the
  fp32 oracle's float64 log-softmax and within 1e-5 (1 + |lse|) of the kernel's own logits.
- test_packed_rows_across_carries: one packed stream at C3 in which followed rows start a new utterance a few steps before a chunk
  boundary; each utterance's next 520 steps meet the same rules against an oracle of that utterance alone, so the packed masks are
  checked against the model, not against the scorer.
- test_prime_from_carried_fronts: C3, a prompt of P = 777 samples scored in four chunks (the fronts of d = 512 reach back past two
  carries, and the last carry of the prompt is 57 pieces of 9 steps), primed, then a teacher-forced continuation of G = 512 steps,
  one launch per step with dumps, on the 8-row cluster, single-CTA latency, tensor-core and fp16 stream kernels: every step's logits
  within the fp16 rule of both oracles forced over [0, P + G), and the last step's xt / skip within 2e-2.  Rows 0 .. 39 are scored
  and primed except on the tensor-core kernel, which primes all B.  A run of fewer than B utterances writes its dumps, and on the
  stream kernel reads its conditioning, at the run's batch stride (DESIGN.md §6), so the test reads and lays those out that way.

The oracle is single-threaded C and its fp16 contract is slow (about 40 ms per C3 step and utterance), so every followed utterance
runs on its own host thread, started with the module's first test, while the GPU works.  On an H100 80GB HBM3 (700 W) with 8 host
CPUs the file ran in about 110 s, with at most 6.1 GiB of device memory in use (l10_b2048).
"""
import os
import re
from concurrent.futures import ThreadPoolExecutor
from functools import lru_cache

import numpy as np
import pytest
import torch

import nv_wavenet_b200 as nw
from oracle import pyoracle as po
from tests import refgen, replay
from tests.test_gpu_parity import _select_fp16_kernel
from tests.test_gpu_zz_prime import _dils, _oracle_trace
from tests.test_gpu_zz_score import _fp16_rule, _log_softmax64

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
A = 256

# case -> (R, S, L, maxDil, engine B, batch_size, N, followed rows)
SCORED = {
    "c3_b64": (64, 256, 20, 512, 64, 64, 1100, (0, 7, 8, 31, 32, 63)),         # edges of the 16-row groups and of the 64-row tiles
    "l10_b2048": (64, 256, 10, 512, 2048, 2048, 565, (0, 15, 1024, 2047)),
    "c3_bs150_of_200": (64, 256, 20, 512, 200, 150, 700, (0, 63, 64, 149)),
    "r128": (128, 256, 12, 256, 128, 128, 600, (0, 63, 127)),
    "r32": (32, 128, 12, 256, 128, 128, 600, (0, 64, 127)),
}
# C3 packed: (R, S, L, maxDil, B, N) and the followed utterances (row, start, length), each starting a few steps before a chunk boundary
PACKED = (64, 256, 20, 512, 64, 1300)
PACKED_UTTS = ((0, 507, 520), (31, 251, 520), (63, 765, 520))
# C3 prime: (R, S, L, maxDil, B, P, G), the followed rows, and the scoring batch_size per kernel (the tensor-core kernel primes all B rows)
PRIME = (64, 256, 20, 512, 64, 777, 512)
PRIME_ROWS = (0, 7, 8, 39)
PRIME_BS = {"lat": 40, "lat_single": 40, "tc": 64, "stream": 40}
PRIME_LAUNCH = {"lat": {"kernel": 18, "cluster": 3, "batch_per_cta": 8}, "lat_single": {"kernel": 18, "cluster": 1},
                "tc": {"kernel": 17}, "stream": {"kernel": 16}}


def score_rows():
    """SCORE_ROWS of wn_engine.cu: the rows (t, b) of one scorer chunk"""
    with open(os.path.join(ROOT, "nv_wavenet_b200", "csrc", "wn_engine.cu")) as f:
        return int(re.search(r"constexpr int SCORE_ROWS = (\d+);", f.read()).group(1))


def chunk_steps(B, N):
    """T of an engine of B utterances and N samples (score_range): min(N, max(1, SCORE_ROWS / B))"""
    return min(N, max(1, score_rows() // B))


def chunks(T, count):
    """(t0, Tc) of the chunks of a call of `count` samples"""
    return [(t0, min(T, count - t0)) for t0 in range(0, count, T)]


def carries_read(t, d, T):
    """carries between the chunk that wrote x_l[t - d] and the one that reads it at step t"""
    return t // T - (t - d) // T


# ------------------------------------------------------------------------------------------------ inputs and the oracle
def _spec(case):
    """(seed, (R, S, A, L, maxDil), oracle steps, followed utterances) of a case"""
    if case in SCORED:
        R, S, L, md, _, _, N, rows = SCORED[case]
        return 3000 + list(SCORED).index(case), (R, S, A, L, md), N, len(rows)
    if case == "packed":
        R, S, L, md = PACKED[:4]
        return 3100, (R, S, A, L, md), PACKED_UTTS[0][2], len(PACKED_UTTS)
    R, S, L, md, _, P, G = PRIME
    return 3200, (R, S, A, L, md), P + G, len(PRIME_ROWS)


@lru_cache(maxsize=None)
def _inputs(case):
    """lively weights, and conditioning [N][L][n][2R] (N(0, 0.5^2)) and selectors [N][n] of the n followed utterances"""
    seed, (R, S, A_, L, _), N, n = _spec(case)
    w = refgen.lively_inputs(seed, R, S, A_, L, 1, 1)
    rng = np.random.default_rng(seed)
    lh = (0.5 * rng.standard_normal((N, L, n, 2 * R), dtype=np.float32)).astype(np.float32)
    return w, lh, rng.random((N, n), dtype=np.float32)


def _utterance(case, i):
    w, lh, sel = _inputs(case)
    v = dict(w)
    v["Lh"], v["selectors"] = np.ascontiguousarray(lh[:, :, i:i + 1]), np.ascontiguousarray(sel[:, i:i + 1])
    return v


def _fp32_run(case, i):
    """the fp32 model's free-running trajectory of followed utterance i and its logits: ([N], [N][A])"""
    _, shape, N, _ = _spec(case)
    y, z32 = replay.oracle_trace(_utterance(case, i), [0], shape, N)
    return y[0], z32[0]


def _fp16_run(case, i, y):
    """the fp16-contract model forced with y: logits [N][A] and its last step's xt [L][R] and skip [L][S]"""
    _, (R, S, A_, L, md), N, _ = _spec(case)
    o, trace = _oracle_trace(_utterance(case, i), L, md, 1, N, y[None], R, S, A_, po.PREC_FP16)
    acts = o.activations()
    return trace[:, 0], acts["xt"][:, 0], acts["skip"][:, 0]


class _Oracles:
    """Every followed utterance of every case on a pool of host threads (the oracle is C, and ctypes releases the GIL while it runs):
    first all fp32 trajectories, then the fp16-contract runs forced with them, in the order the tests ask for them."""

    def __init__(self, cases):
        for c in cases:
            _inputs(c)
        self.pool = ThreadPoolExecutor(max(1, len(os.sched_getaffinity(0))))
        self.runs32 = {(c, i): self.pool.submit(_fp32_run, c, i) for c in cases for i in range(_spec(c)[3])}
        # an fp16 task waits for its trajectory, which is ahead of it in the queue
        self.runs16 = {k: self.pool.submit(lambda k=k: _fp16_run(*k, self.runs32[k].result()[0])) for k in self.runs32}

    def trajectory(self, case):
        """fp32 trajectories [n][N] and logits [n][N][A]"""
        runs = [self.runs32[(case, i)].result() for i in range(_spec(case)[3])]
        return np.stack([r[0] for r in runs]), np.stack([r[1] for r in runs])

    def fp16(self, case):
        """fp16-contract logits [n][N][A], last-step xt [L][n][R] and skip [L][n][S]"""
        runs = [self.runs16[(case, i)].result() for i in range(_spec(case)[3])]
        return np.stack([r[0] for r in runs]), np.stack([r[1] for r in runs], 1), np.stack([r[2] for r in runs], 1)

    def close(self):
        self.pool.shutdown(wait=True, cancel_futures=True)


def _case_of(item):
    if item.originalname == "test_scored_against_the_oracle":
        return item.callspec.params["case"]
    return {"test_packed_rows_across_carries": "packed", "test_prime_from_carried_fronts": "prime"}[item.originalname]


@pytest.fixture(scope="module")
def oracles(request):
    """the oracle runs of the cases this session runs, in its order"""
    o = _Oracles(list(dict.fromkeys(_case_of(i) for i in request.session.items if i.module is request.module)))
    yield o
    o.close()


# ------------------------------------------------------------------------------------------------ helpers (GPU)
def _engine(case, B, N):
    _, (R, S, A_, L, md), _, _ = _spec(case)
    e = nw.NVWavenetInfer(L, md, B, N, nw.AUTO, True, R=R, S=S, A=A_, dtype=nw.FP16)
    e.load(_inputs(case)[0])
    return e


def _conditioning(e, seed, patches):
    """Windows (first, lh [n][L][B][2R]) of the whole conditioning of e: N(0, 0.5^2) drawn on the device, at most 256 MB at a time,
    except that patch (row, t0, v [n][L][2R]) gives row `row` the values v over samples [t0, t0 + n)."""
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    W = max(1, min(e.N, (256 << 20) // (e.L * e.B * 2 * e.R * 4)))
    for first in range(0, e.N, W):
        n = min(W, e.N - first)
        lh = torch.randn((n, e.L, e.B, 2 * e.R), generator=g, device="cuda").mul_(0.5)
        for row, t0, v in patches:
            a, b = max(first, t0), min(first + n, t0 + len(v))
            if a < b:
                lh[a - first:b - first, :, row] = torch.from_numpy(np.ascontiguousarray(v[a - t0:b - t0])).cuda()
        yield first, lh


def _fill_conditioning(e, seed, patches):
    """The whole conditioning store of e, a window at a time through set_conditioning(lh, first, count)"""
    for first, lh in _conditioning(e, seed, patches):
        e.set_conditioning(lh, first, len(lh))
    torch.cuda.synchronize()


def _run_rows(dump, Bs):
    """A dump of a run of Bs utterances read back as [L][B][X]: the run writes it at its own batch stride, [L][Bs][X]"""
    L, _, X = dump.shape
    return dump.reshape(-1)[:L * Bs * X].reshape(L, Bs, X)


def _first_off(z_ref, z):
    """(utterance, step) of the first logit outside the fp16 rule, for the failure message"""
    scale = np.abs(z_ref).max(axis=-1, keepdims=True)
    bad = np.argwhere((np.abs(z - z_ref) > 1e-2 * np.maximum(np.abs(z_ref), 0.25 * scale)).any(axis=-1))
    return tuple(int(v) for v in bad[0]) if bad.size else None


def _rule(z_ref, z, what, mean_rel=None):
    try:
        _fp16_rule(z_ref, z, mean_rel)
    except AssertionError as err:
        raise AssertionError(f"{what}: {err}; first (utterance, step) off the rule: {_first_off(z_ref, z)}") from None


def _check_scores(z16, z32, y, logp, logits, what):
    """the rules of test_oracle_parity_at_every_step at every step: z16, z32, logits [n][T][A]; y, logp [n][T]"""
    assert logits.shape == z32.shape and np.isfinite(logits).all(), what
    _rule(z16, logits, f"{what}, against the fp16 contract", mean_rel=3e-4)
    _rule(z32, logits, f"{what}, against the fp32 model")
    yi = y[..., None].astype(np.int64)
    want = np.take_along_axis(_log_softmax64(z32)[0], yi, -1)[..., 0]
    bad = np.argwhere(np.abs(logp - want) > 2e-2 * np.abs(z32).max(axis=-1))
    assert bad.size == 0, f"{what}: {len(bad)} logp off the fp32 model's; first (utterance, step) {tuple(int(v) for v in bad[0])}"
    own, lse = _log_softmax64(logits)
    own = np.take_along_axis(own, yi, -1)[..., 0]
    bad = np.argwhere(np.abs(logp - own) > 1e-5 * (1 + np.abs(lse)))
    assert bad.size == 0, f"{what}: {len(bad)} logp off the kernel's own logits; first (utterance, step) {tuple(int(v) for v in bad[0])}"


def _mib_in_use(free0):
    return (free0 - torch.cuda.mem_get_info()[0]) / 2**20


# ------------------------------------------------------------------------------------------------ scoring
@pytest.mark.parametrize("case", list(SCORED))
def test_scored_against_the_oracle(case, oracles):
    R, S, L, md, B, bs, N, rows = SCORED[case]
    T, dmax = chunk_steps(B, N), max(_dils(L, md))
    assert dmax >= 2 * T and N - T > dmax and N % T, (case, T, dmax)            # the reach test_score_deep_host.py pins
    y, z32 = oracles.trajectory(case)
    for i, r in enumerate(rows):
        assert len(np.unique(y[i])) > 32, f"{case}: the oracle's row {r} trajectory is degenerate"
    audio = np.random.default_rng(_spec(case)[0]).integers(0, A, (B, N)).astype(np.int32)
    audio[list(rows)] = y
    lh = _inputs(case)[1]

    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    e = _engine(case, B, N)
    _fill_conditioning(e, _spec(case)[0], [(r, 0, lh[:, :, i]) for i, r in enumerate(rows)])
    lp, lg = e.score(torch.from_numpy(audio).cuda(), batch_size=bs, logits=True)
    torch.cuda.synchronize()
    used = _mib_in_use(free0)
    idx = torch.tensor(rows, device="cuda")
    lp, lg = lp[idx].cpu().numpy(), lg[idx].cpu().numpy()
    e.close()
    del e, idx
    torch.cuda.empty_cache()

    z16 = oracles.fp16(case)[0]
    _check_scores(z16, z32, y, lp, lg, f"{case} (B = {B}, batch_size = {bs}, T = {T}) rows {rows}")
    print(f"{case}: B = {B}, batch_size = {bs}, N = {N}, T = {T}, {len(chunks(T, N)) - 1} carries, max d {dmax} in up to "
          f"{-(-dmax // T)} pieces, {used:.0f} MiB of device memory in use")


def test_packed_rows_across_carries(oracles):
    R, S, L, md, B, N = PACKED
    T, dmax = chunk_steps(B, N), max(_dils(L, md))
    y, z32 = oracles.trajectory("packed")
    seed = _spec("packed")[0]
    rng = np.random.default_rng(seed)
    audio = rng.integers(0, A, (B, N)).astype(np.int32)
    starts = np.zeros((B, N), np.uint8)
    for b in range(B):                                          # every row a queue of utterances of 1 to 700 samples
        at = np.cumsum(rng.integers(1, 700, 8))
        starts[b, at[at < N]] = 1
    assert all(n == _spec("packed")[2] for _, _, n in PACKED_UTTS)
    for i, (r, s, n) in enumerate(PACKED_UTTS):
        assert 0 < -s % T <= 8 and n > dmax and carries_read(s + n - 1, dmax, T) >= 2, (r, s, n)
        # the utterance before it starts 300 samples earlier: the fronts of d = 512 hold two utterances' inputs when it starts
        starts[r, max(0, s - 300):s + n] = 0
        starts[r, [max(0, s - 300), s]] = 1
        if s + n < N:
            starts[r, s + n] = 1
        audio[r, s:s + n] = y[i]
    lh = _inputs("packed")[1]
    e = _engine("packed", B, N)
    _fill_conditioning(e, seed, [(r, s, lh[:n, :, i]) for i, (r, s, n) in enumerate(PACKED_UTTS)])
    lp, lg = e.score_stream_packed(audio, starts, 0, logits=True)
    e.close()
    z16 = oracles.fp16("packed")[0]
    for i, (r, s, n) in enumerate(PACKED_UTTS):
        _check_scores(z16[i:i + 1], z32[i:i + 1], y[i:i + 1], lp[r:r + 1, s:s + n], lg[r:r + 1, s:s + n],
                      f"packed C3 (T = {T}), the utterance of row {r} at {s}")


# ------------------------------------------------------------------------------------------------ prime
@pytest.mark.parametrize("kernel", list(PRIME_BS))
def test_prime_from_carried_fronts(kernel, oracles, monkeypatch):
    R, S, L, md, B, P, G = PRIME
    N, Bs, rows = P + G, PRIME_BS[kernel], list(PRIME_ROWS)
    T, dmax = chunk_steps(B, N), max(_dils(L, md))
    assert P > dmax + T and max(rows) < Bs, (P, T)
    _select_fp16_kernel(kernel, monkeypatch)
    y, z32 = oracles.trajectory("prime")
    seed = _spec("prime")[0]
    audio = np.random.default_rng(seed).integers(0, A, (B, N)).astype(np.int32)
    audio[rows] = y
    lh = _inputs("prime")[1]
    e = _engine("prime", B, N)
    patches = [(r, 0, lh[:, :, i]) for i, r in enumerate(rows)]
    _fill_conditioning(e, seed, patches)
    lp, lg = e.score_stream(audio[:Bs, :P], 0, batch_size=Bs, logits=True)
    e.prime_from_score()
    if kernel == "stream" and Bs < B:
        # a run of Bs < B utterances on the stream kernel reads the conditioning store at the run's batch stride (DESIGN.md §6), and
        # the scorer reads the first Bs utterances of the engine's layout: give the continuation its conditioning in the run's layout
        whole = torch.cat([lh_w for _, lh_w in _conditioning(e, seed, patches)])
        store = torch.zeros_like(whole)
        store.view(-1)[:whole[:, :, :Bs].numel()] = whole[:, :, :Bs].reshape(-1)
        e.set_conditioning(store, 0, N)
        torch.cuda.synchronize()
        del whole, store
    e.set_selectors_random(1)
    e.set_forced(audio)
    za = np.empty((len(rows), G, A), np.float32)
    for g in range(G):
        e.run_stream(P + g, 1, Bs, dump_activations=True)
        za[:, g] = e.get_za()[rows]
    info, acts = e.launch_info(), e.activations()
    e.close()
    assert all(info[k] == v for k, v in PRIME_LAUNCH[kernel].items()), info

    z16, xt16, skip16 = oracles.fp16("prime")
    what = f"C3 prime at P = {P} ({kernel}, batch_size {Bs}) rows {rows}"
    _check_scores(z16[:, :P], z32[:, :P], y[:, :P], lp[rows], lg[rows], f"{what}, the prompt")
    _rule(z16[:, P:], za, f"{what}, continuation against the fp16 contract (step P + g)")
    _rule(z32[:, P:], za, f"{what}, continuation against the fp32 model (step P + g)")
    for k, ref in (("xt", xt16), ("skip", skip16)):
        got, sc = _run_rows(acts[k], Bs)[:, rows], np.abs(ref).max()
        assert np.abs(got - ref).max() <= 2e-2 * sc, f"{what}: last step's {k} off by {np.abs(got - ref).max() / sc} of its scale"
