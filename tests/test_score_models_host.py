"""Scoring by model without a GPU: the per-model packed planner, ModelSet's scoring argument checks, the ctypes prototype and
NULL-engine refusal of nvwn_set_score_models, and the C++ facade member."""
import os
import random
import subprocess
import tempfile

import pytest
import torch

import nv_wavenet_b200 as nw
from nv_wavenet_b200 import _lib
from nv_wavenet_b200.nv_wavenet import ModelSet, NVWaveNet, plan_packed, plan_packed_models
from tests.test_models_host import ROOT, _weights


def _queue(seed, n, V, hi=500):
    rng = random.Random(seed)
    return [rng.randint(1, hi) for _ in range(n)], [rng.randrange(V) for _ in range(n)]


@pytest.mark.parametrize("seed,n,V,slots", [(0, 30, 3, 8), (1, 5, 5, 5), (2, 100, 4, 64), (3, 12, 1, 6), (4, 40, 7, 9)])
def test_rows_split_by_samples_and_packed_per_model(seed, n, V, slots):
    lengths, models = _queue(seed, n, V)
    plan, table = plan_packed_models(lengths, models, slots)
    assert (plan, table) == plan_packed_models(lengths, models, slots)              # deterministic
    used = sorted(set(models))
    assert len(table) == slots and table == sorted(table) and sorted(set(table)) == used
    totals = {m: sum(n_ for n_, v in zip(lengths, models) if v == m) for m in used}
    rows = {m: table.count(m) for m in used}
    big = max(used, key=lambda m: (totals[m], -m))
    for m in used:
        share = 1 + (slots - len(used)) * totals[m] // sum(totals.values())
        assert rows[m] == share + (slots - sum(1 + (slots - len(used)) * totals[v] // sum(totals.values()) for v in used)) * (m == big)
    base = {m: table.index(m) for m in used}
    for m in used:
        mine = [u for u in range(n) if models[u] == m]                               # arrival order within the model
        local = plan_packed([lengths[u] for u in mine], rows[m])
        assert [plan[u] for u in mine] == [(base[m] + s, t) for s, t in local]
        assert all(table[plan[u][0]] == m for u in mine)


def test_ties_and_remainders_go_to_the_lower_model():
    plan, table = plan_packed_models([10, 10], [3, 1], 5)
    assert table == [1, 1, 1, 3, 3] and plan == [(3, 0), (0, 0)]
    assert plan_packed_models([1, 1000], [0, 2], 4)[1] == [0, 2, 2, 2]                 # at least one row each


def test_planner_refusals():
    with pytest.raises(ValueError, match="distinct models"):
        plan_packed_models([5, 5, 5], [0, 1, 2], 2)
    for lengths, models in (([5, 0], [0, 1]), ([5], [0, 1]), ([5], [-1]), ([5], [0.5])):
        with pytest.raises(ValueError):
            plan_packed_models(lengths, models, 4)


def test_modelset_scoring_checks_before_any_engine():
    lib = _lib.lib()
    R, S, A = lib.get_R(), lib.get_S(), lib.get_A()
    ms = ModelSet([NVWaveNet(**_weights(R=R, S=S, A=A)), NVWaveNet(**_weights(R=R, S=S, A=A, gen=1))])
    cond, audio = torch.zeros(2 * R, 2, 4, 5), torch.zeros(2, 5, dtype=torch.int32)
    for models, c, a, window in (([0], cond, audio, None), ([0, 2], cond, audio, None), ([0, -1], cond, audio, None),
                                 ([0, 1], cond, audio[:, :4], None), ([0, 1], cond, audio, 0), ([0, 1], cond[:, :, :3], audio, None)):
        with pytest.raises(AssertionError):
            ms.log_likelihood(models, c, a, window=window)
    conds, audios = [torch.zeros(2 * R, 4, 5)] * 2, [torch.zeros(5, dtype=torch.int32)] * 2
    for models, c, a, slots in (([0], conds, audios, 4), ([0, 2], conds, audios, 4), ([0, 1], conds, audios[:1], 4),
                                ([0, 1], conds, [torch.zeros(4, dtype=torch.int32)] * 2, 4), ([0, 1], conds, audios, 0)):
        with pytest.raises(AssertionError):
            ms.log_likelihood_many(models, c, a, slots=slots, window=8)
    with pytest.raises(ValueError, match="distinct models"):
        ms.log_likelihood_many([0, 1], conds, audios, slots=1, window=8)
    for prompts in ([torch.zeros(5, dtype=torch.int32), None], [torch.zeros(2, dtype=torch.int32)], [torch.full((2,), 256), None]):
        with pytest.raises(AssertionError):
            ms.infer_many([0, 1], conds, [1, 2], slots=4, window=8, fp16=True, prompts=prompts)
    with pytest.raises(AssertionError):                                              # prompts need fp16
        ms.infer_many([0, 1], conds, [1, 2], slots=4, window=8, prompts=[torch.zeros(2, dtype=torch.int32), None])
    assert ms._engines == {}
    ms.close()


def test_score_table_entries_that_do_not_fit_a_c_int():
    for bad in ([0, 2 ** 32], [-2 ** 31 - 1], [2 ** 31]):
        with pytest.raises(ValueError):
            nw.NVWavenetInfer.set_score_models(object(), bad)


def test_prototype_and_null_engine():
    lib = _lib.lib()
    fn = lib.nvwn_set_score_models
    assert fn.argtypes is not None and len(fn.argtypes) == 4
    assert lib.nvwn_set_score_models(None, None, 1, None) == -1 and "nvwn_set_score_models" in lib.nvwn_last_error().decode()


def test_cpp_facade_score_models_compiles():
    src = r'''
#include "nv_wavenet.hpp"
int main() {
    typedef nvWavenetInfer<half2, half, 64, 256, 256> W16;
    bool (W16::*table)(const int*, int, cudaStream_t) = &W16::set_score_models;
    int (*c)(nvwn_engine*, const int*, int, void*) = &nvwn_set_score_models;
    (void)table; (void)c;
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
