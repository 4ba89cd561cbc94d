"""Streaming scoring at the C-ABI boundary and in NVWaveNet, without a GPU: the C++ facade's score_stream() compiles (and runs where
a GPU is present), nvwn_score_stream refuses a NULL engine before it needs a device, and the windowed log-likelihood calls refuse
mismatched shapes before they create an engine."""
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


def test_cpp_facade_score_stream_compiles():
    src = r'''
#include "nv_wavenet.hpp"
int main() {
    typedef nvWavenetInfer<half2, half, 64, 256, 256> W16;
    bool (W16::*stream)(const int*, long long, int, int, float*, float*, cudaStream_t) = &W16::score_stream;
    (void)stream;
    if (nvwn_device_count() == 0) return 0;
    W16 w(4, 2, 2, 8);
    int audio[2 * 20];
    float whole[2 * 20], part[2 * 20], logits[2 * 8 * 256];
    for (int i = 0; i < 40; i++) audio[i] = (i * 37) % 256;
    W16 big(4, 2, 2, 20);
    std::vector<float> lh(20 * 4 * 2 * 128, 0.f), sel(20 * 2, 0.5f);
    big.setInputs(lh.data(), sel.data());
    w.setInputs(lh.data(), sel.data());
    if (!big.score(audio, 20, 2, whole)) return 1;
    // the first 8 samples, then samples 8..13 (conditioning 0 everywhere in both engines)
    if (!w.score_stream(audio, 0, 8, 2, part, logits)) return 2;
    for (int b = 0; b < 2; b++) for (int t = 0; t < 8; t++) if (part[b * 8 + t] != whole[b * 20 + t]) return 3;
    int next[2 * 6];
    for (int b = 0; b < 2; b++) for (int t = 0; t < 6; t++) next[b * 6 + t] = audio[b * 20 + 8 + t];
    if (!w.score_stream(next, 8, 6, 2, part)) return 4;
    for (int b = 0; b < 2; b++) for (int t = 0; t < 6; t++) if (part[b * 6 + t] != whole[b * 20 + 8 + t]) return 5;
    if (w.score_stream(next, 13, 6, 2, part)) return 6;                 /* not the next sample */
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


def test_score_stream_null_engine_is_einval():
    lib = _lib.lib()
    audio = (C.c_int * 4)()
    logp = (C.c_float * 4)()
    assert lib.nvwn_score_stream(None, audio, 0, 4, 1, logp, None, None) == -1
    assert b"nvwn_score_stream" in lib.nvwn_last_error()


def _net(L=2):
    lib = _lib.lib()
    R, S, A = lib.get_R(), lib.get_S(), lib.get_A()
    return NVWaveNet(**_weights(L, R, S, A, np.random.default_rng(4))), L, R


def test_log_likelihood_window_rejects_mismatched_shapes_before_any_engine():
    net, L, R = _net()
    cond = torch.zeros(2 * R, 3, L, 10)
    bad = [(cond, torch.zeros(3, 9, dtype=torch.int32), 4),               # audio one sample short
           (cond, torch.zeros(2, 10, dtype=torch.int32), 4),              # audio of another batch
           (torch.zeros(2 * R, 3, L + 1, 10), torch.zeros(3, 10, dtype=torch.int32), 4),
           (cond, torch.zeros(3, 10, dtype=torch.int32), 0)]              # no window
    for c, a, w in bad:
        with pytest.raises(AssertionError):
            net.log_likelihood(c, a, window=w)
    assert net.engines_created == 0


def test_log_likelihood_from_features_rejects_mismatched_shapes_before_any_engine():
    net, L, R = _net()
    Cc, K, stride, B, T = 5, 8, 4, 3, 6
    z = lambda *s: torch.zeros(s)
    good = dict(upsample_weight=z(Cc, Cc, K), upsample_bias=z(Cc), cond_weight=z(L * 2 * R, Cc), cond_bias=z(L * 2 * R), stride=stride)
    frames, audio = z(B, Cc, T), torch.zeros(B, T * stride, dtype=torch.int32)
    bad = [(frames, audio[:, 1:], good),                                  # audio not T * stride samples
           (frames, audio[1:], good),                                     # audio of another batch
           (z(B, Cc + 1, T), audio, good),                                # frames of another channel count
           (z(Cc, T), audio, good),                                       # frames not [B][C][T]
           (z(B, Cc, 0), audio[:, :0], good),                             # no frames
           (frames, audio, dict(good, upsample_weight=z(Cc, Cc + 1, K))),
           (frames, audio, dict(good, upsample_bias=z(Cc + 1))),
           (frames, audio, dict(good, cond_weight=z(L * 2 * R + 1, Cc))),
           (frames, audio, dict(good, cond_bias=z(L * R))),
           (frames, audio, dict(good, stride=K + 1))]                     # window < stride
    for window in (None, 8):
        for f, a, kw in bad:
            with pytest.raises(AssertionError):
                net.log_likelihood_from_features(f, a, window=window, **kw)
    with pytest.raises(AssertionError):
        net.log_likelihood_from_features(frames, audio, window=0, **good)
    assert net.engines_created == 0
