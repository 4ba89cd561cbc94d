"""Prompted continuous batching at the C-ABI boundary and in NVWaveNet, without a GPU: the C++ facade's prime_slots_from_score()
compiles (and runs where a GPU is present), nvwn_prime_slots_from_score refuses a NULL engine before it needs a device, and
infer_many(prompts=...) refuses bad prompts before it creates an engine."""
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


def test_cpp_facade_prime_slots_from_score_compiles():
    src = r'''
#include "nv_wavenet.hpp"
int main() {
    typedef nvWavenetInfer<half2, half, 64, 256, 256> W16;
    bool (W16::*prime)(const int*, const int*, int, const unsigned long long*, cudaStream_t) = &W16::prime_slots_from_score;
    (void)prime;
    if (nvwn_device_count() == 0) return 0;
    W16 w(4, 2, 3, 8);
    std::vector<float> lh(8 * 4 * 3 * 128, 0.f), sel(8 * 3, 0.5f);
    w.setInputs(lh.data(), sel.data());
    int rows[1] = {1}, slots[1] = {2};
    unsigned long long seeds[1] = {7};
    if (w.prime_slots_from_score(rows, slots, 1, seeds)) return 1;       /* nothing scored yet */
    int audio[2 * 3] = {1, 2, 3, 4, 5, 6};
    float logp[2 * 3];
    if (!w.score_stream(audio, 0, 3, 2, logp)) return 2;
    if (!w.prime_slots_from_score(rows, slots, 1, seeds)) return 3;
    if (!w.run_stream(0, 5, 3)) return 4;                               /* slot 2 continues row 1 from sample 3 of its own */
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


def test_prime_slots_null_engine_is_einval():
    lib = _lib.lib()
    assert lib.nvwn_prime_slots_from_score(None, None, None, 0, None, None) == -1
    assert b"nvwn_prime_slots_from_score" in lib.nvwn_last_error()


def test_infer_many_prompts_rejected_before_any_engine():
    net, L, R = _net()
    lengths = [10, 12]
    conds = [torch.zeros(2 * R, L, n) for n in lengths]
    good = torch.zeros(4, dtype=torch.int32)
    bad = [dict(prompts=[good]),                                            # one prompt for two utterances
           dict(prompts=[torch.zeros(1, 4, dtype=torch.int32), None]),     # not [P]
           dict(prompts=[torch.zeros(0, dtype=torch.int32), None]),        # P = 0
           dict(prompts=[None, torch.zeros(12, dtype=torch.int32)]),       # P = samples: nothing to generate
           dict(prompts=[torch.zeros(11, dtype=torch.int32), None]),       # P > samples
           dict(prompts=[torch.zeros(4), None]),                           # float codes
           dict(prompts=[np.zeros(4, np.float64), None]),
           dict(prompts=[torch.zeros(4, dtype=torch.bool), None]),
           dict(prompts=[torch.full((4,), 256, dtype=torch.int32), None]), # codes outside [0, A)
           dict(prompts=[torch.full((4,), -1, dtype=torch.int32), None]),
           dict(prompts=[good, None], fp16=False)]                        # the scorer is fp16
    for kw in bad:
        kw = dict(dict(fp16=True), **kw)
        with pytest.raises(AssertionError):
            net.infer_many(conds, [1, 2], slots=2, window=8, **kw)
    assert net.engines_created == 0
