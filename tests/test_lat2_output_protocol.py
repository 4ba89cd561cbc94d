"""Protocol model of the cluster kernel's output layers (tools/lat2_protocol_model.py): the prep CTA's half of Zs / Za must run in
its step loop between shipping step (t + 1, 1) and waiting for the buffer of step (t + 1, NAP + 1), and each CTA must wait for the
peer's relu(Zs) half before it reads OB1.  Each mutation re-introduces one of those defects and the model must see it."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import lat2_protocol_model as m  # noqa: E402


def _hits(n, **kw):
    hits, last = 0, None
    for s in range(n):
        try:
            m.trial(s, **kw)
        except m.Hazard as e:
            hits, last = hits + 1, str(e)
    return hits, last


def test_long_runs_with_a_slow_output_half_are_clean():
    for slow in ({"prep.w6": 10.0}, {"tail.w3": 10.0}, {"prep.w1": 0.3}):
        sim = m.trial(5, L=12, T=5, slow=slow, max_dil=4)
        assert all(p.done for p in sim.procs)


def test_mutation_prep_output_half_after_the_tile_buffer_wait_deadlocks():
    hits, msg = _hits(3, bug="prep_out_late", L=12, T=2)
    assert hits == 3 and msg.startswith("deadlock"), msg


def test_mutation_reading_ob1_before_the_peer_half_lands():
    hits, msg = _hits(6, bug="no_ob1full_wait", L=12, T=2)
    assert hits >= 1 and ".ob1" in msg, msg
