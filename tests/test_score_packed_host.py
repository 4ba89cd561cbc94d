"""Packed scoring without a GPU: the plan_packed schedule, the window assembly of log_likelihood_many (segments, start flags and
padding) against restatements, the argument checks of the queue calls, and the declarations of nvwn_score_stream_packed."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import nv_wavenet_b200 as nw
from nv_wavenet_b200 import _lib
from nv_wavenet_b200.nv_wavenet import _pack_window, _packed_windows, plan_packed
from tests.test_score_stream_host import _net

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _brute_plan(lengths, slots):
    """plan_packed restated: utterance u goes to the row, lowest first among equals, whose utterances so far end earliest."""
    plan = []
    for n in lengths:
        end = lambda s: sum(lengths[v] for v, (r, _) in enumerate(plan) if r == s)
        best = min(range(slots), key=lambda s: (end(s), s))
        plan.append((best, end(best)))
    return plan


@pytest.mark.parametrize("seed", range(6))
def test_plan_packed_properties(seed):
    rng = np.random.default_rng(seed)
    slots = int(rng.integers(1, 9))
    lengths = [int(v) for v in rng.integers(1, 60, int(rng.integers(0, 40)))]
    if seed == 0:
        lengths = [5] * 7                                                # every choice a tie
    plan = plan_packed(lengths, slots)
    assert plan == _brute_plan(lengths, slots)
    for s in range(slots):
        mine = [(start, lengths[u], u) for u, (r, start) in enumerate(plan) if r == s]
        assert [u for _, _, u in mine] == sorted(u for _, _, u in mine)            # arrival order within a row
        assert all(a + n == b for (a, n, _), (b, _, _) in zip(mine, mine[1:]))    # end to end, no overlap, no gap
        assert not mine or mine[0][0] == 0
    if seed == 0:
        assert plan[:min(slots, 7)] == [(s, 0) for s in range(min(slots, 7))]       # ties go to the lowest row


def test_plan_packed_rejects_bad_arguments():
    for lengths, slots in (([3, 0, 2], 2), ([-1], 1), ([4], 0), ([4], -3)):
        with pytest.raises(ValueError):
            plan_packed(lengths, slots)
    assert plan_packed([], 3) == []


@pytest.mark.parametrize("window", [1, 2, 5, 16, 64, 1000])
def test_window_assembly(window):
    rng = np.random.default_rng(window)
    slots = 4
    lengths = [int(v) for v in rng.integers(1, 40, 13)]
    plan = plan_packed(lengths, slots)
    audios = [torch.from_numpy(rng.integers(0, 256, n).astype(np.int32)) for n in lengths]
    end = max(s + n for (_, s), n in zip(plan, lengths))
    # the whole stream restated: row s holds its utterances end to end, then code 128
    stream = np.full((slots, end), 128, np.int32)
    flags = np.zeros((slots, end), np.uint8)
    for u, (s, start) in enumerate(plan):
        stream[s, start:start + lengths[u]] = audios[u].numpy()
        flags[s, start] = 1
    windows = _packed_windows(plan, lengths, window)
    assert [(f, n) for f, n, _ in windows] == [(f, min(window, end - f)) for f in range(0, end, window)]
    seen = [0] * len(lengths)
    for first, count, segs in windows:
        keys = [(s, o) for s, _, _, o, _ in segs]
        assert keys == sorted(keys)                                        # by row, then time
        for s, u, a, o, m in segs:
            assert plan[u][0] == s and m >= 1 and 0 <= o and o + m <= count
            assert plan[u][1] + a == first + o and a + m <= lengths[u]
            assert a == seen[u]                                           # each utterance's samples once, in order
            seen[u] += m
        audio, starts = _pack_window(count, segs, audios, slots)
        assert audio.dtype == torch.int32 and starts.dtype == torch.uint8
        assert np.array_equal(audio.numpy(), stream[:, first:first + count])
        assert np.array_equal(starts.numpy(), flags[:, first:first + count])
    assert seen == lengths


def test_queue_calls_reject_bad_arguments_before_any_engine():
    net, L, R = _net()
    conds = [torch.zeros(2 * R, L, n) for n in (5, 3)]
    auds = [torch.zeros(n, dtype=torch.int32) for n in (5, 3)]
    bad = [(conds, auds[:1], {}),                                         # one audio short
           (conds, [auds[0], torch.zeros(4, dtype=torch.int32)], {}),      # audio of another length
           ([torch.zeros(2 * R, L + 1, 5)], auds[:1], {}),                 # another layer count
           ([torch.zeros(2 * R, L, 0)], [torch.zeros(0, dtype=torch.int32)], {}),
           (conds, auds, {"slots": 0}), (conds, auds, {"window": 0}), (conds, auds, {"window": None})]
    for c, a, kw in bad:
        with pytest.raises(AssertionError):
            net.log_likelihood_many(c, a, **kw)
    Cc, K, stride = 5, 8, 4
    z = lambda *s: torch.zeros(s)
    good = dict(upsample_weight=z(Cc, Cc, K), upsample_bias=z(Cc), cond_weight=z(L * 2 * R, Cc), cond_bias=z(L * 2 * R), stride=stride)
    frames = [z(Cc, 3), z(Cc, 2)]
    for f, a, kw in ((frames, [torch.zeros(12), torch.zeros(7)], {}), ([z(Cc + 1, 3)], [torch.zeros(12)], {}), ([z(Cc, 0)], [torch.zeros(0)], {}),
                     (frames, [torch.zeros(12), torch.zeros(8)], {"slots": 0}), (frames, [torch.zeros(12), torch.zeros(8)], dict(good, stride=K + 1))):
        with pytest.raises(AssertionError):
            net.log_likelihood_many_from_features(f, a, **dict(good, **kw))
    assert net.engines_created == 0


def test_declarations():
    hdr = open(os.path.join(ROOT, "include", "nvwn_b200.h")).read()
    m = re.search(r"int nvwn_score_stream_packed\(([^)]*)\);", hdr)
    assert m, "nvwn_b200.h does not declare nvwn_score_stream_packed"
    c_args = [re.sub(r"\s+", " ", a.strip()) for a in m.group(1).split(",")]
    assert c_args == ["nvwn_engine* e", "const int* audio", "const unsigned char* starts", "long long first_sample", "int count",
                      "int batch_size", "float* logp", "float* logits", "void* stream"]


def test_null_engine_is_einval():
    lib = _lib.lib()
    audio, starts, logp = (C.c_int * 4)(), (C.c_ubyte * 4)(), (C.c_float * 4)()
    assert lib.nvwn_score_stream_packed(None, audio, starts, 0, 4, 1, logp, None, None) == -1
    assert b"nvwn_score_stream_packed" in lib.nvwn_last_error()


def test_cpp_facade_score_stream_packed_compiles():
    """The facade's score_stream_packed and the C declaration have the same arguments."""
    src = r'''
#include "nv_wavenet.hpp"
int main() {
    typedef nvWavenetInfer<half2, half, 64, 256, 256> W16;
    bool (W16::*packed)(const int*, const unsigned char*, long long, int, int, float*, float*, cudaStream_t) = &W16::score_stream_packed;
    int (*abi)(nvwn_engine*, const int*, const unsigned char*, long long, int, int, float*, float*, void*) = &nvwn_score_stream_packed;
    (void)packed; (void)abi;
    return 0;
}
'''
    with tempfile.TemporaryDirectory() as d:
        f = os.path.join(d, "t.cpp")
        open(f, "w").write(src)
        cmd = ["g++", "-std=c++14", "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include", f, "-o", os.path.join(d, "t"),
               "-L", os.path.dirname(nw.LIB_PATH), "-lwavenet_infer", "-Wl,-rpath," + os.path.dirname(nw.LIB_PATH)]
        res = subprocess.run(cmd, capture_output=True, text=True)
        assert res.returncode == 0, res.stderr
