"""Multi-model serving without a GPU: the slot planner with models and groups, the window tables, ModelSet's argument checks, the
ctypes prototypes and the C++ facade members."""
import os
import random
import subprocess
import tempfile

import pytest
import torch

import nv_wavenet_b200 as nw
from nv_wavenet_b200 import _lib
from nv_wavenet_b200.nv_wavenet import ModelSet, NVWaveNet, _windows, group_models, plan_slots

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _one_model_plan(lengths, slots, window):
    """The one-model schedule, written the way it always was: each utterance to the lowest free slot at the first boundary."""
    ends, plan, t = [0] * slots, [], 0
    for n in lengths:
        while True:
            free = [s for s in range(slots) if ends[s] <= t]
            if free:
                break
            t = (min(ends) + window - 1) // window * window
        plan.append((free[0], t))
        ends[free[0]] = t + n
    return plan


def _queue(seed, n, V, lo=1, hi=60):
    rng = random.Random(seed)
    return [rng.randint(lo, hi) for _ in range(n)], [rng.randrange(V) for _ in range(n)]


CASES = [(seed, slots, group, window, V) for seed, (slots, group, window, V) in
         enumerate([(8, 4, 7, 3), (10, 4, 5, 2), (16, 8, 16, 4), (5, 2, 3, 3), (64, 8, 13, 8), (7, 16, 4, 2), (12, 1, 6, 5)])]


@pytest.mark.parametrize("seed,slots,group,window,V", CASES)
def test_group_runs_its_model_for_every_span(seed, slots, group, window, V):
    lengths, models = _queue(seed, 40, V)
    plan = plan_slots(lengths, slots, window, models, group)
    assert all(p is not None for p in plan)
    for u, (s, t) in enumerate(plan):
        assert 0 <= s < slots and t % window == 0
        for v, (s2, t2) in enumerate(plan):
            overlap = t < t2 + lengths[v] and t2 < t + lengths[u]
            if v != u and overlap and s2 // group == s // group:
                assert models[v] == models[u], (u, v)            # a group runs one model while any of its utterances is live
            if v != u and overlap:
                assert s2 != s, (u, v)                           # no slot holds two utterances at once


@pytest.mark.parametrize("seed,slots,group,window,V", CASES)
def test_window_tables_match_the_plan(seed, slots, group, window, V):
    lengths, models = _queue(seed, 30, V)
    plan = plan_slots(lengths, slots, window, models, group)
    for first, count, _, live in _windows(plan, lengths, window):
        table = group_models(plan, lengths, models, first, count, group, slots)
        assert len(table) == (slots + group - 1) // group
        for s, u, _, _ in live:
            assert table[s // group] == models[u]
        idle = {g for g in range(len(table))} - {s // group for s, _, _, _ in live}
        assert all(table[g] == 0 for g in idle)


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("group", [1, 4, 8])
def test_one_model_plan_is_unchanged(seed, group):
    rng = random.Random(100 + seed)
    lengths = [rng.randint(1, 90) for _ in range(rng.randint(1, 50))]
    slots, window = rng.randint(1, 12), rng.randint(1, 20)
    want = _one_model_plan(lengths, slots, window)
    assert plan_slots(lengths, slots, window) == want
    assert plan_slots(lengths, slots, window, [0] * len(lengths), group) == want
    assert plan_slots(lengths, slots, window, [3] * len(lengths), group) == want


def test_plan_is_deterministic_and_keeps_arrival_order_per_model():
    lengths, models = _queue(7, 60, 4)
    a = plan_slots(lengths, 16, 9, models, 4)
    assert a == plan_slots(list(lengths), 16, 9, list(models), 4)
    for m in range(4):
        starts = [a[u][1] for u in range(len(lengths)) if models[u] == m]
        assert starts == sorted(starts)                          # a model's utterances start in arrival order


def test_idle_group_takes_the_earliest_waiting_model():
    # two groups of two slots: model 1 waits behind model 0's utterances and gets the second group at once
    plan = plan_slots([10, 10, 10, 10], 4, 5, [0, 0, 1, 0], 2)
    # utterance 3 (model 0) may not take slot 3 of group 1, which runs model 1 while utterance 2 lives there: it waits for a
    # slot of group 0
    assert plan == [(0, 0), (1, 0), (2, 0), (0, 10)]


@pytest.mark.parametrize("args", [
    dict(lengths=[3, 4], slots=4, window=2, models=[0], group=2),          # one model per utterance
    dict(lengths=[3, 4], slots=4, window=2, models=[0, -1], group=2),      # negative index
    dict(lengths=[3, 4], slots=4, window=2, models=[0, 1.5], group=2),     # not an index
    dict(lengths=[3, 4], slots=4, window=2, models=[0, 1], group=0),       # empty groups
    dict(lengths=[3, 0], slots=4, window=2, models=[0, 1], group=2),       # empty utterance
    dict(lengths=[3, 4], slots=0, window=2, models=[0, 1], group=2),
    dict(lengths=[3, 4], slots=4, window=0, models=[0, 1], group=2),
])
def test_bad_plan_arguments(args):
    with pytest.raises(ValueError):
        plan_slots(**args)


def _weights(L=4, R=64, S=256, A=256, md=2, tanh=True, gen=0):
    g = torch.Generator().manual_seed(gen)
    r = lambda *s: torch.randn(*s, generator=g) * 0.1
    return dict(embedding_prev=r(A, R), embedding_curr=r(A, R), conv_out_weight=r(A, S, 1), conv_end_weight=r(A, A, 1),
                dilate_weights=[r(2 * R, R, 2) for _ in range(L)], dilate_biases=[r(2 * R) for _ in range(L)], max_dilation=md,
                res_weights=[r(R, R, 1) for _ in range(L - 1)], res_biases=[r(R) for _ in range(L - 1)],
                skip_weights=[r(S, R, 1) for _ in range(L)], skip_biases=[r(S) for _ in range(L)], use_embed_tanh=tanh)


def test_modelset_checks_before_any_engine():
    lib = _lib.lib()
    R, S, A = lib.get_R(), lib.get_S(), lib.get_A()
    a, b = NVWaveNet(**_weights(R=R, S=S, A=A)), NVWaveNet(**_weights(R=R, S=S, A=A, gen=1))
    for nets in ([], [a, NVWaveNet(**_weights(L=5, R=R, S=S, A=A))], [a, NVWaveNet(**_weights(R=R, S=S, A=A, md=4))],
                 [a, NVWaveNet(**_weights(R=R, S=S, A=A, tanh=False))], [a] * (nw.infer.MAX_MODELS + 1)):
        with pytest.raises(AssertionError):
            ModelSet(nets)
    ms = ModelSet([a, b])
    cond = [torch.zeros(2 * R, 4, 5)]
    for models, conds, seeds in (([2], cond, [1]), ([-1], cond, [1]), ([0, 1], cond, [1]), ([0], cond, [1, 2]),
                                 ([0], [torch.zeros(2 * R, 3, 5)], [1])):
        with pytest.raises(AssertionError):
            ms.infer_many(models, conds, seeds, slots=4, window=8)
    assert ms._engines == {}
    ms.close()


def test_group_table_entries_that_do_not_fit_a_c_int():
    # checked before the engine is touched: an entry of 2**32 would otherwise wrap to model 0
    for bad in ([0, 2 ** 32], [-2 ** 31 - 1], [2 ** 31]):
        with pytest.raises(ValueError):
            nw.NVWavenetInfer.set_group_models(object(), bad)


def test_plan_of_a_long_one_model_queue():
    lengths = [1 + (u * 7919) % 500 for u in range(20000)]
    assert plan_slots(lengths, 64, 256, [0] * len(lengths), 8) == _one_model_plan(lengths, 64, 256)


def test_prototypes_and_null_engine():
    lib = _lib.lib()
    for name, n in (("nvwn_set_model", 3), ("nvwn_model_group", 2), ("nvwn_set_group_models", 4)):
        fn = getattr(lib, name)
        assert fn.argtypes is not None and len(fn.argtypes) == n
    assert lib.nvwn_set_model(None, 1, None) == -1 and "nvwn_set_model" in lib.nvwn_last_error().decode()
    assert lib.nvwn_model_group(None, None) == -1 and "nvwn_model_group" in lib.nvwn_last_error().decode()
    assert lib.nvwn_set_group_models(None, None, 1, None) == -1 and "nvwn_set_group_models" in lib.nvwn_last_error().decode()
    assert _lib.MAX_MODELS == 64


def test_cpp_facade_model_members_compile():
    src = r'''
#include "nv_wavenet.hpp"
int main() {
    typedef nvWavenetInfer<half2, half, 64, 256, 256> W16;
    bool (W16::*set)(int, const W16&) = &W16::set_model;
    int (W16::*group)() = &W16::model_group;
    bool (W16::*table)(const int*, int, cudaStream_t) = &W16::set_group_models;
    int (*c1)(nvwn_engine*, int, const nvwn_engine*) = &nvwn_set_model;
    int (*c2)(nvwn_engine*, int*) = &nvwn_model_group;
    int (*c3)(nvwn_engine*, const int*, int, void*) = &nvwn_set_group_models;
    static_assert(NVWN_MAX_MODELS == 64, "models per engine");
    (void)set; (void)group; (void)table; (void)c1; (void)c2; (void)c3;
    return 0;
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
