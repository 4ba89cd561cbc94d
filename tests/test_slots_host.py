"""CPU checks of continuous batching: the schedule of NVWaveNet.infer_many (plan_slots), the C++ facade's per-slot members, and the
per-slot entry points' refusal of a NULL engine."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import nv_wavenet_b200 as nw
from nv_wavenet_b200 import _lib
from nv_wavenet_b200.nv_wavenet import plan_slots

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _check_plan(lengths, slots, window):
    plan = plan_slots(lengths, slots, window)
    assert len(plan) == len(lengths)                                  # each utterance in exactly one slot
    starts = [t for _, t in plan]
    assert all(0 <= s < slots for s, _ in plan)
    assert all(t % window == 0 for t in starts)                       # restarts only at window boundaries
    assert starts == sorted(starts)                                   # FIFO: no utterance starts before an earlier arrival
    by_slot = {}
    for (s, t), n in zip(plan, lengths):
        by_slot.setdefault(s, []).append((t, t + n))
    for spans in by_slot.values():                                    # never two utterances at once in one slot
        spans.sort()
        assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))
    # no idle wait: an utterance that starts after its predecessor found every slot busy at the boundary before its start
    for u in range(1, len(plan)):
        t = plan[u][1]
        if t > plan[u - 1][1]:
            prev = t - window
            busy = {s2 for (s2, t2), n2 in zip(plan[:u], lengths[:u]) if t2 <= prev < t2 + n2}
            assert len(busy) == slots, (u, t, busy)
    return plan


@pytest.mark.parametrize("lengths, slots, window", [
    ([1, 5, 37, 513, 700, 1300, 2049], 3, 512),
    ([10] * 9, 3, 10),                           # ends exactly at a boundary: the slot is free at that boundary
    ([11] * 9, 3, 10),                           # ends one sample past it: the slot waits a whole window
    ([4000], 64, 4096),
    (list(range(1, 40)), 1, 7),                  # one slot: strictly one after another
])
def test_plan_slots_examples(lengths, slots, window):
    _check_plan(lengths, slots, window)


def test_plan_slots_first_fit_details():
    assert plan_slots([10] * 4, 3, 10) == [(0, 0), (1, 0), (2, 0), (0, 10)]
    assert plan_slots([11, 3, 30, 5], 2, 10) == [(0, 0), (1, 0), (1, 10), (0, 20)]
    assert plan_slots([], 4, 8) == []


def test_plan_slots_random_mixes():
    rng = np.random.default_rng(5)
    for _ in range(40):
        slots, window = int(rng.integers(1, 9)), int(rng.integers(1, 50))
        lengths = [int(v) for v in rng.integers(1, 200, int(rng.integers(1, 60)))]
        _check_plan(lengths, slots, window)


@pytest.mark.parametrize("args", [([0, 1], 0, 4), ([1], 2, 0), ([3, 0], 2, 4)])
def test_plan_slots_rejects(args):
    with pytest.raises(ValueError):
        plan_slots(*args)


def test_null_engine_is_einval():
    lib = _lib.lib()
    slots = (C.c_int * 1)(0)
    lh = (C.c_float * 256)()
    calls = {"nvwn_restart_slots": lambda: lib.nvwn_restart_slots(None, slots, 1, None, None),
             "nvwn_set_conditioning_slots": lambda: lib.nvwn_set_conditioning_slots(None, lh, slots, 1, 0, 1, None),
             "nvwn_set_selectors_random_slots": lambda: lib.nvwn_set_selectors_random_slots(None, 0, 1, None)}
    for name, call in calls.items():
        assert call() == -1
        assert name in lib.nvwn_last_error().decode()


def test_cpp_facade_slot_members_compile():
    src = r'''
#include "nv_wavenet.hpp"
int main() {
    typedef nvWavenetInfer<float, float, 64, 256, 256> W32;
    typedef nvWavenetInfer<half2, half, 64, 256, 256> W16;
    bool (W16::*restart)(const int*, int, const unsigned long long*, cudaStream_t) = &W16::restart_slots;
    bool (W16::*cond)(const float*, const int*, int, long long, int, cudaStream_t) = &W16::set_conditioning_slots;
    bool (W32::*sel)(long long, int, cudaStream_t) = &W32::set_selectors_random_slots;
    (void)restart; (void)cond; (void)sel;
    if (nvwn_device_count() == 0) return 0;
    W32 w(2, 2, 3, 4);
    const int slots[2] = {2, 0};
    const unsigned long long seeds[2] = {7, 8};
    const int twice[2] = {1, 1};
    return w.restart_slots(slots, 2, seeds) && w.set_selectors_random_slots(0, 4) && !w.restart_slots(twice, 2) ? 0 : 1;
}
'''
    with tempfile.TemporaryDirectory() as d:
        f = os.path.join(d, "t.cpp")
        open(f, "w").write(src)
        exe = os.path.join(d, "t")
        cmd = ["g++", "-std=c++14", "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include", f, "-o", exe,
               "-L", os.path.dirname(nw.LIB_PATH), "-lwavenet_infer", "-Wl,-rpath," + os.path.dirname(nw.LIB_PATH)]
        res = subprocess.run(cmd, capture_output=True, text=True)
        assert res.returncode == 0, res.stderr
        assert subprocess.run([exe], capture_output=True).returncode == 0
