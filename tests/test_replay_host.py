"""The replay check of tests/replay.py on the CPU: it accepts the oracle's own trajectories and rejects each kind of slip a
kernel could make, without a GPU."""
import numpy as np
import pytest

from oracle import pyoracle as po
from tests import refgen, replay

R, S, A, L, MD, B, N = 64, 256, 256, 6, 8, 4, 80              # ring of 9 slots: it wraps 8 times
PEAK = 8.0                                                    # six layers need a larger Wza than L16 for a mean max-probability ~0.45


@pytest.fixture(scope="module")
def run():
    w = refgen.export_inputs(3, R, S, A, L, B, N, peak=PEAK)
    y, z = replay.oracle_trace(w, range(B), (R, S, A, L, MD), N, tanh_embed=False)
    return w, y, z


def _replay(w, y, delta=replay.DELTA, sel=None, tanh_embed=False):
    """Replays trajectory y of all B utterances through the fp32 oracle and checks it."""
    _, z = replay.oracle_trace(w, range(B), (R, S, A, L, MD), N, forced=y, tanh_embed=tanh_embed)
    return replay.check(y, z, w["selectors"] if sel is None else sel, delta, replay.MAX_AMBIGUOUS)


def test_windows_by_hand():
    cdf = np.array([[0.1, 0.5, 0.5, 1.0]])
    assert [int(v[0]) for v in replay.windows(cdf, [0.5], 0.0)] == [3, 3]        # the first class whose CDF exceeds 0.5
    assert [int(v[0]) for v in replay.windows(cdf, [0.3], 0.25)] == [0, 3]
    assert [int(v[0]) for v in replay.windows(cdf, [0.05], 0.0)] == [0, 0]
    assert [int(v[0]) for v in replay.windows(cdf, [0.9999], 0.01)] == [3, 3]     # past the last boundary: the last class


def test_export_inputs_are_the_exported_configuration(run):
    w, y, z = run
    assert not w["embPrev"].any() and not w["Bzs"].any() and not w["Bza"].any()
    assert not w["Wres"][L - 1].any() and not w["Bres"][L - 1].any() and w["Wres"][L - 2].any()
    assert 0.8 < w["embCur"].std() < 1.2
    p = np.diff(replay.cdf64(z), axis=-1, prepend=0.0)
    assert 0.3 < p.max(axis=-1).mean() < 0.6                    # peaked, as a trained model's distribution is
    assert len(np.unique(y)) > 32


def test_fp32_trajectory_replays_exactly(run):
    w, y, _ = run
    assert _replay(w, y, delta=0.0) == 0.0


def test_fp16_contract_trajectory_within_delta(run):
    """The PREC_FP16 oracle stands in for an fp16 kernel: its own free-running trajectory, a different one from the fp32
    model's, replays against the fp32 oracle at the delta the GPU tests use."""
    w, y32, _ = run
    y16, _ = replay.oracle_trace(w, range(B), (R, S, A, L, MD), N, tanh_embed=False, prec=po.PREC_FP16)
    assert not np.array_equal(y16, y32)
    _, z16 = replay.oracle_trace(w, range(B), (R, S, A, L, MD), N, forced=y32, tanh_embed=False, prec=po.PREC_FP16)
    _, z32 = replay.oracle_trace(w, range(B), (R, S, A, L, MD), N, forced=y32, tanh_embed=False)
    assert replay.cdf_deviation(z32, z16) < replay.DELTA / 2
    assert 0.0 < _replay(w, y16) <= replay.MAX_AMBIGUOUS


def test_one_changed_sample_fails(run):
    w, y, z = run
    lo, hi = replay.windows(replay.cdf64(z), w["selectors"].T, replay.DELTA)
    b, t = np.argwhere(lo == hi)[len(np.argwhere(lo == hi)) // 2]
    bad = y.copy()
    bad[b, t] = (bad[b, t] + 1) % A
    with pytest.raises(AssertionError, match=rf"of {B * N} sampled indices outside their window; first: row {b} step {t}:"):
        _replay(w, bad)


def test_trajectory_one_step_late_fails(run):
    w, y, _ = run
    late = y.copy()
    late[:, 1:] = y[:, :-1]
    with pytest.raises(AssertionError, match="sampled indices outside their window"):
        _replay(w, late)


def test_neighbouring_selectors_fail(run):
    w, y, _ = run
    with pytest.raises(AssertionError, match="sampled indices outside their window"):
        _replay(w, y, sel=np.ascontiguousarray(w["selectors"][:, [1, 2, 3, 0]]))


def test_embedding_tanh_in_the_replay_fails(run):
    w, y, _ = run
    with pytest.raises(AssertionError, match="sampled indices outside their window"):
        _replay(w, y, tanh_embed=True)


def test_large_delta_fails_the_ambiguity_bound(run):
    w, y, _ = run
    with pytest.raises(AssertionError, match="ambiguous fraction"):
        _replay(w, y, delta=0.05)
