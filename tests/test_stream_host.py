"""CPU checks of streaming generation: the splitting of absolute sample ranges at the wrap of the ring buffers, and the C++ facade's
run_stream against the C-ABI."""
import os
import subprocess
import tempfile

import pytest

import nv_wavenet_b200 as nw
from nv_wavenet_b200.infer import split_at_wrap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("first, count, N, want", [
    (0, 8, 8, [(0, 0, 8)]),                     # fits exactly
    (16, 8, 8, [(0, 0, 8)]),                    # fits exactly, a later lap
    (5, 3, 8, [(5, 0, 3)]),                     # ends at the wrap
    (8, 3, 8, [(0, 0, 3)]),                     # starts at the wrap
    (13, 6, 8, [(5, 0, 3), (0, 3, 3)]),         # crosses it
    (7, 8, 8, [(7, 0, 1), (0, 1, 7)]),          # a whole ring, crossing it
    (3, 0, 8, []),
    (10 ** 12 + 1, 2, 4, [(1, 0, 2)]),          # absolute times past 32 bits
])
def test_split_at_wrap(first, count, N, want):
    pieces = split_at_wrap(first, count, N)
    assert pieces == want
    covered = [first + off + j for _, off, n in pieces for j in range(n)]
    assert covered == list(range(first, first + count))
    assert all(pos + n <= N for pos, _, n in pieces)
    assert [(first + off) % N for pos, off, _ in pieces] == [pos for pos, _, _ in pieces]


@pytest.mark.parametrize("first, count", [(-1, 1), (0, -1), (0, 9)])
def test_split_at_wrap_rejects(first, count):
    with pytest.raises(ValueError):
        split_at_wrap(first, count, 8)


def test_cpp_facade_run_stream_compiles():
    src = r'''
#include "nv_wavenet.hpp"
int main() {
    typedef nvWavenetInfer<float, float, 64, 256, 256> W32;
    typedef nvWavenetInfer<half2, half, 64, 256, 256> W16;
    bool (W16::*stream_fn)(long long, int, int, bool, cudaStream_t) = &W16::run_stream;
    (void)stream_fn;
    if (nvwn_device_count() == 0) return 0;
    W32 w(2, 2, 1, 4);
    return w.run_stream(0, 4, 1) && w.run_stream(4, 3, 1) && !w.run_stream(3, 1, 1) ? 0 : 1;
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
