"""Protocol model of the three-CTA cluster kernel (tools/lat2_protocol_model.py), chain CTA's weight ring: in 8-row clusters the
compute warps read the Wcur fragments of step n + 1 behind the h barrier of step n, so the sync warp waits for ring piece n + 1
before that barrier instead of for piece n before the x barrier (16-row clusters keep the latter).  With two or three ring slots,
either tile height, random latencies and a slow producer nothing deadlocks and no slot is rewritten before its last reader;
dropping the early wait, or handing a piece back before its Wres fragments are read, is seen by the model."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import lat2_protocol_model as m  # noqa: E402


@pytest.mark.parametrize("nslot0", [2, 3])
@pytest.mark.parametrize("seed", range(12))
def test_random_trials(seed, nslot0):
    sim = m.trial(seed, nslot0=nslot0, wcur_ahead=True)
    assert all(p.done for p in sim.procs)


@pytest.mark.parametrize("slow", [{"chain.producer": 3.0}, {"chain.producer": 10.0}, {"chain.producer": 10.0, "chain.sync": 3.0},
                                  {"chain.producer": 0.3, "chain.w5": 3.0}])
@pytest.mark.parametrize("nslot0", [2, 3])
@pytest.mark.parametrize("rows", [8, 16])
def test_a_slow_producer_only_slows_the_chain(slow, nslot0, rows):
    sim = m.trial(4, L=12, T=3, slow=slow, max_dil=4, rows=rows, nslot0=nslot0, wcur_ahead=True)
    assert all(p.done for p in sim.procs)
    assert sim.min_history_margin is not None and sim.min_history_margin >= 3, sim.min_history_margin


def _hits(n, **kw):
    hits, last = 0, None
    for s in range(n):
        try:
            m.trial(s, **kw)
        except m.Hazard as e:
            hits, last = hits + 1, str(e)
    return hits, last


@pytest.mark.parametrize("nslot0", [2, 3])
def test_mutation_sync_warp_does_not_wait_for_the_next_piece(nslot0):
    """Without the wait for piece n + 1 before the h barrier of step n, the compute warps read its Wcur fragments before it landed."""
    hits, msg = _hits(4, bug="no_early_full_wait", L=12, T=2, slow={"chain.producer": 10.0}, nslot0=nslot0, wcur_ahead=True)
    assert hits == 4 and "in cring" in msg and "expects 0 " not in msg, msg


@pytest.mark.parametrize("nslot0", [2, 3])
def test_mutation_piece_handed_back_before_its_res_fragments_are_read(nslot0):
    """The empty arrival for piece n stays behind the h barrier of step n: the Wres fragments are read under the gate."""
    hits, msg = _hits(8, bug="empty_early", L=12, T=2, slow={"chain.w3": 10.0}, nslot0=nslot0, wcur_ahead=True)
    assert hits >= 1 and msg.startswith("cring") and "overwritten" in msg, msg


@pytest.mark.parametrize("nslot0", [2, 3])
def test_wcur_behind_the_x_barrier(nslot0):
    """Wcur read behind the x barrier, piece n waited for before it: the 16-row clusters' protocol."""
    sim = m.trial(5, L=12, T=3, nslot0=nslot0, wcur_ahead=False, slow={"chain.producer": 10.0})
    assert all(p.done for p in sim.procs)
    hits, msg = _hits(4, bug="no_full_wait", L=12, T=2, slow={"chain.producer": 10.0}, nslot0=nslot0, wcur_ahead=False)
    assert hits == 4 and "in cring" in msg, msg


def test_the_defaults_follow_the_kernel():
    assert (m.Sim(rows=8).wcur_ahead, m.Sim(rows=8).nslot0) == (True, 3)
    assert (m.Sim(rows=16).wcur_ahead, m.Sim(rows=16).nslot0) == (False, 2)
