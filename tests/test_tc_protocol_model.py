"""The synchronisation protocol of a warp-specialised fused tensor-core schedule, checked on the CPU by a discrete-event
model (tools/tc_protocol_model.py): random latencies, stressed roles, every layer / dilation / dump / buffering variant.
Three protocol defects (a single conditioning buffer, a commit with nothing outstanding, phase aliasing) are
re-introduced to show the model sees them."""
import random

import pytest

from tools import tc_protocol_model as M


def dilations(L, md):
    out, d = [], 1
    for _ in range(L):
        out.append(d)
        d = d * 2 if d * 2 <= md else 1
    return out


@pytest.mark.parametrize("seed", range(40))
def test_randomised_schedules_complete_without_hazard(seed):
    rng = random.Random(seed)
    L = rng.choice([1, 2, 3, 5, 20])
    kw = dict(L=L, S=rng.choice([128, 256]), NC=rng.choice([1, 2]), steps=rng.choice([2, 3]), dil=dilations(L, rng.choice([1, 2, 4, 8, 512])),
              dump_last=rng.random() < 0.4, t0=rng.choice([0, 1, 7, 600]),
              slow=rng.choice([None, {"B": 4.0}, {"A": 3.0}, {"C": 5.0}, {"E": 3.0}, {"P": 6.0}, {"B": 0.3, "E": 0.3}]))
    sim = M.trial(seed, **kw)
    assert {"P", "A", "B", "C"} <= sim.finished and not sim.late_commits


def test_c3_shape_all_layers_with_history():
    sim = M.trial(7, L=20, S=256, NC=2, steps=2, dil=dilations(20, 512), t0=600)
    assert len(sim.finished) >= 12


def _first_hazard(bug, tries, **kw):
    for seed in range(tries):
        try:
            M.trial(seed, bug=bug, **kw)
        except M.Hazard as h:
            return str(h)
    return None


def test_model_sees_the_single_buffer_conditioning_deadlock():
    h = _first_hazard("cond_first", 3, L=5, NC=1, steps=2, dil=dilations(5, 4))
    assert h and "deadlock" in h


def test_model_sees_a_commit_with_nothing_outstanding():
    h = _first_hazard("empty_commit", 3, L=5, steps=2, dil=dilations(5, 512))
    assert h and "no MMA of this thread in flight" in h


def test_model_sees_phase_aliasing_on_a_single_b_done_barrier():
    # the signalling role finishes an iteration before the waiter has looked at the previous one
    h = _first_hazard("one_b_done", 200, L=20, steps=2, dil=dilations(20, 512), slow={"B": 0.2, "E": 3.0})
    assert h and ("aliasing" in h or "deadlock" in h)


def test_model_sees_phase_aliasing_on_a_single_tile_published_barrier():
    # role B a whole gate behind role A: two completions past the one it waits for
    h = _first_hazard("one_epi_done", 1, L=20, S=128, NC=2, steps=3, dil=[1] * 20, dump_last=True, t0=1, slow={"C": 0.5, "B": 8})
    assert h is None or "aliasing" in h or "deadlock" in h
    hs = [_first_hazard("one_epi_done", 60, L=20, S=128, steps=3, dil=[1] * 20, dump_last=True, t0=1, slow={"B": 8})]
    assert any(x and ("aliasing" in x or "deadlock" in x) for x in hs)


@pytest.mark.parametrize("seed", range(20))
def test_unfused_schedule_completes_without_hazard(seed):
    rng = random.Random(1000 + seed)
    L = rng.choice([1, 2, 3, 5, 20])
    kw = dict(L=L, S=rng.choice([128, 256]), NC=rng.choice([1, 2]), nstage=rng.choice([3, 4, 6, 8]), steps=rng.choice([2, 3]),
              dil=dilations(L, rng.choice([1, 2, 8, 512])), t0=rng.choice([0, 1, 7, 600]),
              slow=rng.choice([None, {"A": 4.0}, {"E": 3.0}, {"P": 6.0}, {"E": 0.3}]))
    sim = M.trial(seed, schedule="unfused", **kw)
    assert {"P", "A"} <= sim.finished
