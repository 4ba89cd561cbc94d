"""Teacher-forced scoring at the C-ABI boundary, without a GPU: the C++ facade's score() compiles (and runs where a GPU is
present), and nvwn_score validates its arguments before it needs a device."""
import ctypes as C
import os
import subprocess
import tempfile

import nv_wavenet_b200 as nw
from nv_wavenet_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cpp_facade_score_compiles():
    src = r'''
#include "nv_wavenet.hpp"
int main() {
    typedef nvWavenetInfer<half2, half, 64, 256, 256> W16;
    if (nvwn_device_count() == 0) return 0;
    W16 w(4, 2, 2, 8);
    int audio[16];
    float logp[16], logits[16 * 256];
    for (int i = 0; i < 16; i++) audio[i] = (i * 37) % 256;
    if (!w.score(audio, 8, 2, logp)) return 1;
    if (!w.score(audio, 8, 2, logp, logits)) return 2;
    for (int i = 0; i < 16; i++) if (!(logp[i] <= 0.f)) return 3;
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
        assert subprocess.run([exe]).returncode == 0


def test_score_null_engine_is_einval():
    lib = _lib.lib()
    audio = (C.c_int * 4)()
    logp = (C.c_float * 4)()
    assert lib.nvwn_score(None, audio, 4, 1, logp, None, None) == -1
    assert b"nvwn_score" in lib.nvwn_last_error()
