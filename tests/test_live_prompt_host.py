"""CPU checks of prompted live streams: when a prompt becomes scoreable, how the prompts of one step are grouped into scoring streams, a
LivePool with prompted streams driven through recording engines (scoring pieces, saved states, resumes from sample P), argument checks
before any engine exists, the ctypes prototype and the C++ facade's new member."""
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import nv_wavenet_b200 as nw
from nv_wavenet_b200 import _lib
from nv_wavenet_b200.infer import live_frames
from nv_wavenet_b200.nv_wavenet import LivePool, NVWaveNet, plan_prompt_groups, prompt_frames
from tests.test_live_pool_host import _PoolEngine
from tests.test_nv_wavenet_py import _weights

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_prompt_frames_is_the_last_frame_the_prompt_reads():
    for K, stride in [(12, 5), (800, 200), (4, 4), (7, 3)]:
        for P in range(1, 60):
            assert prompt_frames(P, stride) == live_frames(0, P, K, stride)[1], (K, stride, P)


def test_prompt_groups():
    assert plan_prompt_groups([], 4) == []
    assert plan_prompt_groups([(3, 40), (1, 7), (9, 7), (2, 13)], 4) == [[(1, 7), (9, 7), (2, 13), (3, 40)]]
    assert plan_prompt_groups([(0, 5), (1, 3), (2, 9)], 2) == [[(1, 3), (0, 5)], [(2, 9)]]


class _Scorer:
    """a scoring engine that records its calls and checks the scoring stream's rules; a state is [position, seed]"""

    def __init__(self, B, N):
        self.B, self.N, self.calls, self.next = B, N, [], None

    def cond_producer_load(self, feats, *net):
        assert feats.shape[0] == self.B
        self.frames = feats.shape[2]
        self.calls.append(("load", feats.shape[2]))

    def cond_producer_run_stream(self, a, m):
        assert 1 <= m <= self.N and a // self.N == (a + m - 1) // self.N and (a + m) <= self.frames * self.stride
        self.produced = (a, m)

    def score_stream(self, codes, a):
        assert self.produced == (a, codes.shape[1]) and (a == 0 or a == self.next)
        self.next = a + codes.shape[1]
        self.calls.append(("score", a, codes.shape[1], codes.shape[0]))

    def score_save_states(self, rows, seeds):
        self.calls.append(("save", list(rows), self.next))
        return torch.tensor([[self.next, s] for s in seeds], dtype=torch.int64)

    def close(self):
        pass


def _pool(B=3, W=10, K=12, stride=5, scorer_rows=None):
    eng = _PoolEngine(B, W, K, stride)
    eng.dtype, eng.A = _lib.FP16, 256
    sc = _Scorer(scorer_rows or B, W)
    sc.stride = stride
    pool = LivePool(eng, 2, K, stride, scorer=lambda: sc, network=tuple(np.zeros(1, np.float32) for _ in range(4)))
    pool.device = "cpu"
    return pool, eng, sc


def test_prompted_pool_against_recording_engines():
    """Prompts of 23 and 9 samples become scoreable in one step and share a scoring stream, rows by length, scored in pieces that end
    at 9, at the window and at 23; a prompt of 14 whose frames arrive over several steps is scored in the step its third frame
    arrives; a prompt of 40 whose frames never cover it ends with nothing.  Each prompted stream's outputs are its samples P, P + 1,
    ... in order; it resumes with start t - P from the first frame sample P reads."""
    K, stride, W = 12, 5, 10
    pool, eng, sc = _pool(3, W, K, stride)
    p = lambda P: torch.full((P,), 7, dtype=torch.int32)
    ids = [pool.open(1), pool.open(2, p(23)), pool.open(3, p(9)), pool.open(4, p(14)), pool.open(5, p(40))]
    totals = [8, 12, 6, 9, 5]
    got, given = {}, [0] * 5
    script = {0: [2, 5, 2, 1, 2], 1: [2, 0, 0, 1, 1], 2: [2, 2, 2, 1, 2], 3: [1, 3, 2, 2, 0]}     # frames per stream per step
    for step in range(60):
        for j, i in enumerate(ids):
            k = min(script.get(step, [2] * 5)[j], totals[j] - given[j])
            if k:
                pool.push(i, np.zeros((2, k), np.float32))
                given[j] += k
            elif given[j] == totals[j] and i in pool._streams and not pool._streams[i].finished:
                pool.finish(i)
        n_calls = len(sc.calls)
        for i, y in pool.step().items():
            got.setdefault(i, []).append(y)
        new = sc.calls[n_calls:]
        if step == 0:
            # streams 1 and 2 hold 5 and 2 frames: prompts of 23 (5 frames) and 9 (2 frames), one stream, rows by length
            assert new == [("load", 5), ("score", 0, 9, 2), ("save", [0], 9), ("score", 9, 1, 2), ("score", 10, 10, 2),
                           ("score", 20, 3, 2), ("save", [1], 23)], new
        elif step == 1:
            assert new == [], "stream 3 holds 2 of the 3 frames its prompt reads"
        elif step == 2:
            assert new == [("load", 3), ("score", 0, 10, 1), ("score", 10, 4, 1), ("save", [0], 14)], new
        else:
            assert new == [], new
        if not pool._streams:
            break
    assert not pool._streams and ids[4] not in got
    for j, P in [(0, 0), (1, 23), (2, 9), (3, 14)]:
        y = torch.cat(got[ids[j]])
        assert torch.equal(y, torch.arange(P, totals[j] * stride, dtype=torch.int32)), (j, y)
    loads = [c for c in eng.calls if c[0] == "load"]
    assert {9, 14, 23} <= {p for c in loads for p in c[2]}                 # each prompted stream resumes from its P (others from parks)
    for k, c in enumerate(eng.calls):
        if c[0] == "load":
            att = next(a for a in eng.calls[k + 1:] if a[0] == "attach")
            run = next(r for r in eng.calls[k:] if r[0] == "run")
            for b, P in zip(c[1], c[2]):
                j = att[1].index(b)
                assert att[2][j] == run[1] - P and att[3][j] == live_frames(P, 1, K, stride)[0]


def test_prompt_groups_split_at_the_scoring_rows():
    pool, eng, sc = _pool(3, 10, 12, 5, scorer_rows=2)
    for P in (4, 9, 2):
        pool.open(P, torch.full((P,), 1, dtype=torch.int32))
    for i in range(3):
        pool.push(i, np.zeros((2, 2), np.float32))
    pool.step()
    assert [c for c in sc.calls if c[0] == "save"] == [("save", [0], 4), ("save", [1], 9), ("save", [0], 2)]


def test_a_prompt_and_nothing_after_it_leaves_the_pool():
    pool, eng, sc = _pool()
    i = pool.open(1, torch.full((10,), 3, dtype=torch.int32))
    pool.push(i, np.zeros((2, 2), np.float32))
    pool.finish(i)
    assert pool.step() == {} and not pool._streams and eng.calls == [] and [c[0] for c in sc.calls][-1] == "save"


def test_pool_prompt_checks():
    pool, eng, sc = _pool()
    for bad in (torch.zeros(0, dtype=torch.int32), torch.full((3,), 256, dtype=torch.int32), torch.zeros(3), torch.zeros((2, 3), dtype=torch.int32)):
        with pytest.raises(AssertionError):
            pool.open(1, bad)
    eng.dtype = _lib.FP32
    with pytest.raises(AssertionError, match="fp16"):
        pool.open(1, torch.zeros(3, dtype=torch.int32))
    bare = LivePool(_PoolEngine(2, 10, 12, 5), 2, 12, 5)
    bare._eng.dtype, bare._eng.A = _lib.FP16, 256
    with pytest.raises(AssertionError, match="no scoring engine"):
        bare.open(1, torch.zeros(3, dtype=torch.int32))
    assert not pool._streams and not bare._streams and sc.calls == []


def test_open_live_prompt_checks_before_any_engine(monkeypatch):
    lib = _lib.lib()
    R, S, A = lib.get_R(), lib.get_S(), lib.get_A()
    L, Cc, K, stride = 2, 5, 8, 4
    net = NVWaveNet(**_weights(L, R, S, A, np.random.default_rng(5)))
    made = []
    monkeypatch.setattr(net, "_new_engine", lambda *a: made.append(a))
    z = lambda *s: torch.zeros(s)
    good = dict(upsample_weight=z(Cc, Cc, K), upsample_bias=z(Cc), cond_weight=z(L * 2 * R, Cc), cond_bias=z(L * 2 * R), stride=stride,
                batch_size=2, seed=1, window=8, fp16=True)
    for kw in [dict(good, prompt=torch.zeros((3, 4), dtype=torch.int32)), dict(good, prompt=torch.zeros((2, 0), dtype=torch.int32)),
               dict(good, prompt=torch.full((2, 4), A, dtype=torch.int32)), dict(good, prompt=torch.zeros((2, 4))),
               dict(good, fp16=False, prompt=torch.zeros((2, 4), dtype=torch.int32))]:
        with pytest.raises(AssertionError):
            net.open_live(**kw)
    assert made == []


def test_prototype_and_null_engine():
    lib = _lib.lib()
    assert lib.nvwn_score_save_states.argtypes is not None and len(lib.nvwn_score_save_states.argtypes) == 6
    assert lib.nvwn_score_save_states(None, None, 1, None, None, None) == -1
    assert "nvwn_score_save_states" in lib.nvwn_last_error().decode()


def test_cpp_facade_score_save_states_compiles():
    src = r'''
#include "nv_wavenet.hpp"
int main() {
    typedef nvWavenetInfer<half2, half, 64, 256, 256> W16;
    bool (W16::*save)(const int*, int, const unsigned long long*, void*, cudaStream_t) = &W16::score_save_states;
    int (*c)(nvwn_engine*, const int*, int, const unsigned long long*, void*, void*) = &nvwn_score_save_states;
    (void)save; (void)c;
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
