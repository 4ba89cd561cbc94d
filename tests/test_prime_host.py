"""Prompted generation at the C-ABI boundary and in NVWaveNet, without a GPU: the C++ facade's prime_from_score() compiles (and runs
where a GPU is present), nvwn_prime_from_score refuses a NULL engine before it needs a device, and infer() refuses a bad prompt or
window before it creates an engine."""
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import nv_wavenet_b200 as nw
from nv_wavenet_b200 import _lib
from tests.test_score_stream_host import _net

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cpp_facade_prime_from_score_compiles():
    src = r'''
#include "nv_wavenet.hpp"
int main() {
    typedef nvWavenetInfer<half2, half, 64, 256, 256> W16;
    bool (W16::*prime)(cudaStream_t) = &W16::prime_from_score;
    (void)prime;
    if (nvwn_device_count() == 0) return 0;
    W16 w(4, 2, 2, 8);
    std::vector<float> lh(8 * 4 * 2 * 128, 0.f), sel(8 * 2, 0.5f);
    w.setInputs(lh.data(), sel.data());
    if (w.prime_from_score()) return 1;                                 /* nothing scored yet */
    int audio[2 * 3] = {1, 2, 3, 4, 5, 6};
    float logp[2 * 3];
    if (!w.score_stream(audio, 0, 3, 2, logp)) return 2;
    if (!w.prime_from_score()) return 3;
    if (!w.run_stream(3, 5, 2)) return 4;                               /* the continuation of samples [3, 8) */
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


def test_prime_null_engine_is_einval():
    lib = _lib.lib()
    assert lib.nvwn_prime_from_score(None, None) == -1
    assert b"nvwn_prime_from_score" in lib.nvwn_last_error()


def test_infer_prompt_rejects_bad_prompts_before_any_engine():
    net, L, R = _net()
    B, T = 3, 10
    cond = torch.zeros(2 * R, B, L, T)
    good = torch.zeros(B, 4, dtype=torch.int32)
    bad = [dict(prompt=torch.zeros(B, dtype=torch.int32)),                 # not [batch][P]
           dict(prompt=torch.zeros(B - 1, 4, dtype=torch.int32)),         # another batch
           dict(prompt=torch.zeros(B, 0, dtype=torch.int32)),             # P = 0
           dict(prompt=torch.zeros(B, T, dtype=torch.int32)),             # P = samples: nothing to generate
           dict(prompt=torch.zeros(B, T + 1, dtype=torch.int32)),
           dict(prompt=torch.zeros(B, 4)),                                # float codes
           dict(prompt=np.zeros((B, 4), np.float64)),
           dict(prompt=torch.zeros(B, 4, dtype=torch.bool)),
           dict(prompt=torch.full((B, 4), 256, dtype=torch.int32)),       # codes outside [0, A)
           dict(prompt=torch.full((B, 4), -1, dtype=torch.int32)),
           dict(prompt=good, fp16=False),                                 # the scorer is fp16
           dict(prompt=good, window=0),
           dict(prompt=None, window=0),                                   # the window rule holds without a prompt too
           dict(prompt=None, window=0, fp16=False)]
    for kw in bad:
        kw = dict(fp16=True, seed=1, **kw) if "fp16" not in kw else dict(seed=1, **kw)
        with pytest.raises(AssertionError):
            net.infer(cond, 0, **kw)
    assert net.engines_created == 0
