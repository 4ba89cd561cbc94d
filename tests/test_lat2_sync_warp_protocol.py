"""Protocol model of the three-CTA cluster kernel (tools/lat2_protocol_model.py), chain CTA's sync warp: the compute warps of the
chain CTA wait on no mbarrier in the layer loop; the sync warp waits for them, enters their named barrier behind what it saw
land and hands the buffers they have read back.  A slow sync warp only slows the cluster, and removing any one of its
handshakes is seen by the model."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import lat2_protocol_model as m  # noqa: E402


@pytest.mark.parametrize("slow", [{"chain.sync": 10.0}, {"chain.sync": 0.3}, {"chain.sync": 3.0, "tail.w3": 3.0}])
@pytest.mark.parametrize("rows", [8, 16])
def test_a_slow_sync_warp_only_slows_the_others(slow, rows):
    sim = m.trial(3, L=12, T=3, slow=slow, max_dil=4, rows=rows)
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


def test_mutation_sync_warp_does_not_wait_for_the_weight_piece():
    hits, msg = _hits(4, bug="no_full_wait", L=12, T=2, slow={"chain.producer": 10.0})
    assert hits == 4 and "in cring" in msg, msg


def test_mutation_sync_warp_does_not_wait_for_the_pre_activation_tile():
    hits, msg = _hits(4, bug="no_apfull_wait", L=12, T=2, slow={"prep.producer": 10.0})
    assert hits == 4 and "in ap" in msg, msg


def test_mutation_sync_warp_never_frees_the_weight_slot():
    hits, msg = _hits(3, bug="no_empty", L=12, T=2)
    assert hits == 3 and msg.startswith("deadlock") and "chain.producer" in msg, msg


def test_mutation_sync_warp_waits_for_the_h_buffer_behind_the_x_barrier():
    """The compute warps send h tile n right after the x barrier of step n: the wait for the tail's buffer must come before it."""
    hits, msg = _hits(6, bug="hfree_late", L=12, T=2, slow={"tail.w3": 10.0})
    assert hits >= 1 and msg.startswith("h") and "overwritten" in msg, msg
