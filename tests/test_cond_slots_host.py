"""CPU checks of the per-slot conditioning producer: the C++ facade's members, the entry points' refusal of a NULL engine, and
NVWaveNet.infer_many_from_features refusing mismatched shapes before it creates an engine."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import nv_wavenet_b200 as nw
from nv_wavenet_b200 import _lib
from nv_wavenet_b200.nv_wavenet import NVWaveNet
from tests.test_nv_wavenet_py import _weights

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_null_engine_is_einval():
    lib = _lib.lib()
    slots = (C.c_int * 1)(0)
    frames = (C.c_float * 8)()
    ptrs = (C.c_void_p * 1)(C.addressof(frames))
    count = (C.c_int * 1)(2)
    start = (C.c_longlong * 1)(0)
    calls = {"nvwn_cond_producer_set_weights": lambda: lib.nvwn_cond_producer_set_weights(None, 2, frames, frames, 4, 2, frames, frames, None),
             "nvwn_cond_producer_set_slots": lambda: lib.nvwn_cond_producer_set_slots(None, slots, 1, ptrs, count, start, None),
             "nvwn_cond_producer_run_slots": lambda: lib.nvwn_cond_producer_run_slots(None, slots, 1, 0, 1, None)}
    for name, call in calls.items():
        assert call() == -1
        assert name in lib.nvwn_last_error().decode()


def test_cpp_facade_producer_members_compile():
    src = r'''
#include "nv_wavenet.hpp"
int main() {
    typedef nvWavenetInfer<float, float, 64, 256, 256> W32;
    typedef nvWavenetInfer<half2, half, 64, 256, 256> W16;
    bool (W16::*weights)(int, const float*, const float*, int, int, const float*, const float*, cudaStream_t) = &W16::cond_producer_set_weights;
    bool (W16::*attach)(const int*, int, const float* const*, const int*, const long long*, cudaStream_t) = &W16::cond_producer_set_slots;
    bool (W32::*run)(const int*, int, long long, int, cudaStream_t) = &W32::cond_producer_run_slots;
    (void)weights; (void)attach; (void)run;
    if (nvwn_device_count() == 0) return 0;
    W32 w(2, 2, 3, 8);
    const int C = 2, K = 4, stride = 2, LR = 2 * 2 * 64;
    std::vector<float> wu(C * C * K, 0.5f), bu(C, 0.1f), wc(LR * C, 0.25f), bc(LR, 0.f), frames(C * 3, 1.f);
    const float* f[2] = {frames.data(), frames.data()};
    const int slots[2] = {2, 0}, counts[2] = {3, 1};
    const long long starts[2] = {0, 2};
    return w.cond_producer_set_weights(C, wu.data(), bu.data(), K, stride, wc.data(), bc.data()) && w.cond_producer_set_slots(slots, 2, f, counts, starts) &&
           w.cond_producer_run_slots(slots, 2, 2, 6) && !w.cond_producer_run_slots(slots, 2, 1, 6) ? 0 : 1;
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


def test_infer_many_from_features_rejects_mismatched_shapes_before_any_engine():
    lib = _lib.lib()
    R, S, A = lib.get_R(), lib.get_S(), lib.get_A()
    L, Cc, K, stride = 2, 5, 8, 4
    net = NVWaveNet(**_weights(L, R, S, A, np.random.default_rng(3)))
    z = lambda *s: torch.zeros(s)
    good = dict(upsample_weight=z(Cc, Cc, K), upsample_bias=z(Cc), cond_weight=z(L * 2 * R, Cc), cond_bias=z(L * 2 * R), stride=stride)
    frames = [z(Cc, 3), z(Cc, 1)]
    bad = [(frames, [1], good),                                                   # one seed short
           ([z(Cc + 1, 3)], [1], good),                                           # frames of another channel count
           ([z(Cc, 3, 1)], [1], good),                                            # frames not [C][T]
           ([z(Cc, 0)], [1], good),                                               # no frames
           (frames, [1, 2], dict(good, upsample_weight=z(Cc, Cc + 1, K))),
           (frames, [1, 2], dict(good, upsample_bias=z(Cc + 1))),
           (frames, [1, 2], dict(good, cond_weight=z(L * 2 * R + 1, Cc))),
           (frames, [1, 2], dict(good, cond_weight=z(L * 2 * R, Cc - 1))),
           (frames, [1, 2], dict(good, cond_bias=z(L * R))),
           (frames, [1, 2], dict(good, stride=K + 1))]                            # window < stride
    for f, seeds, kw in bad:
        with pytest.raises(AssertionError):
            net.infer_many_from_features(f, seeds, slots=2, window=8, **kw)
    assert net.engines_created == 0
