"""Replay check: every sampled index of a generation run against the CPU oracle's distribution at that step.

A run records its sampled index at every step, teacher-forced or not, and the oracle does the same when it is given a forced
history.  So a trajectory y that a kernel produced (or the history it was forced with) is replayed through the fp32 oracle
as its forced input; the oracle's logits at step t are then the model's distribution given exactly the history the kernel
saw, and y[b][t] must be the class the selector picks from it.  The kernel computes that distribution in its own arithmetic,
so a selector within delta of a CDF boundary may fall on either side; every other step must match exactly.

Rows are independent utterances, so the oracle follows only the rows it is given (a list of utterance indices, chosen to
cover tile positions), not a prefix of the batch.
"""
import numpy as np

from oracle import pyoracle as po

# delta and the bound on the ambiguous fraction for peaked distributions (refgen.export_inputs, mean max-probability ~0.45).
# There the fp16-contract oracle and every fp16 kernel keep the CDF within about 2e-3 of the fp32 oracle's (measured in
# tests/test_gpu_zz_replay.py); delta is about three times that, and leaves 14-21 % of the steps ambiguous.
DELTA, MAX_AMBIGUOUS = 6e-3, 0.35


def sub_rows(w, rows):
    """The inputs of utterances `rows` (conditioning and selectors sliced on their batch axis)."""
    v = dict(w)
    v["Lh"] = np.ascontiguousarray(w["Lh"][:, :, rows])
    v["selectors"] = np.ascontiguousarray(w["selectors"][:, rows])
    return v


def oracle_trace(w, rows, shape, N, forced=None, tanh_embed=True, prec=po.PREC_FP32):
    """The oracle (MATH_PORTABLE) on utterances `rows` of inputs w for N steps, forced with `forced` [len(rows)][N] (None:
    free-running).  shape = (R, S, A, L, maxDil).  Returns (its sampled indices [len(rows)][N], logits [len(rows)][N][A])."""
    R, S, A, L, md = shape
    rows = list(rows)
    Bo = len(rows)
    v = sub_rows(w, rows)
    v["Lh"] = np.ascontiguousarray(v["Lh"][:N])
    v["selectors"] = np.ascontiguousarray(v["selectors"][:N])
    o = po.Oracle(L, Bo, N, R, S, A, md, math=po.MATH_PORTABLE, prec=prec, tanh_embed=tanh_embed)
    o.load(v)
    o.set_inputs(v["Lh"], v["selectors"])
    if forced is not None:
        o.set_forced(np.ascontiguousarray(np.asarray(forced)[:, :N], np.int32))
    trace = np.zeros((N, Bo, A), np.float32)
    o.set_logit_trace(trace)
    y = o.run(N, Bo)
    return y, np.ascontiguousarray(trace.transpose(1, 0, 2))


def cdf64(logits):
    """Cumulative softmax in float64, along the last axis."""
    z = np.asarray(logits, np.float64)
    p = np.exp(z - z.max(axis=-1, keepdims=True))
    cs = np.cumsum(p, axis=-1)
    return cs / cs[..., -1:]


def windows(cdf, sel, delta):
    """[lo, hi] per step: lo the first class whose CDF exceeds sel - delta, hi the first whose CDF exceeds sel + delta (the
    last class if none does).  cdf [..., A], sel [...]."""
    A = cdf.shape[-1]
    sel = np.asarray(sel, np.float64)[..., None]
    lo = np.minimum((cdf <= sel - delta).sum(axis=-1), A - 1)
    hi = np.minimum((cdf <= sel + delta).sum(axis=-1), A - 1)
    return lo, hi


def check(y, logits, sel, delta, max_ambiguous, start=0, what=""):
    """Every y[b][t], t >= start, lies in its window from the oracle's logits [b][t][A] and the selectors sel [t][b], and is
    exactly the window's class wherever the window holds one class.  Asserts that the fraction of steps whose window holds
    more than one class is at most max_ambiguous (so a large delta cannot make the check vacuous) and returns it."""
    y = np.asarray(y)[:, start:]
    logits = np.asarray(logits)[:, start:]
    sel = np.asarray(sel).T[:, start:]                      # [b][t]
    assert y.shape == sel.shape == logits.shape[:2], (y.shape, sel.shape, logits.shape)
    lo, hi = windows(cdf64(logits), sel, delta)
    bad = np.argwhere((y < lo) | (y > hi))
    if bad.size:
        b, t = bad[0]
        raise AssertionError(f"{what}{len(bad)} of {y.size} sampled indices outside their window; first: row {b} step "
                             f"{t + start}: sampled {y[b, t]}, window [{lo[b, t]}, {hi[b, t]}], selector {sel[b, t]}")
    ambiguous = float((lo != hi).mean())
    assert ambiguous <= max_ambiguous, f"{what}ambiguous fraction {ambiguous:.3f} > {max_ambiguous} (delta {delta})"
    return ambiguous


def cdf_deviation(logits_ref, logits):
    """max |CDF(logits) - CDF(logits_ref)| over every class and step."""
    return float(np.abs(cdf64(logits) - cdf64(logits_ref)).max())
