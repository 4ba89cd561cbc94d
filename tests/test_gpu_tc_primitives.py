"""Pins the wgmma building blocks of the tensor-core kernel on real hardware: K-major SWIZZLE_128B operand
tiles written row-per-thread, pre-tiled weight images moved by 1-D bulk TMA, shared-memory descriptors,
K-slice and row-block advance, accumulate flag, the accumulator fragment layout.  Checked against numpy."""
import ctypes as C

import numpy as np
import pytest

from nv_wavenet_b200 import _lib

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("N,K,mode", [(128, 64, 0), (128, 128, 0), (64, 64, 0), (256, 64, 0), (256, 256, 0), (256, 128, 1), (128, 256, 1)])
def test_umma_gemm_matches_numpy(N, K, mode):
    lib = _lib.lib()
    fn = lib.nvwn_selftest_umma
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int]
    rng = np.random.default_rng(N + K)
    A = rng.standard_normal((128, K)).astype(np.float16)
    B = rng.standard_normal((N, K)).astype(np.float16)
    D = np.zeros((128, N), np.float32)
    assert fn(A.ctypes.data, B.ctypes.data, N, K, D.ctypes.data, mode) == 0
    ref = A.astype(np.float32) @ B.astype(np.float32).T
    err = np.abs(D - ref).max()
    assert err < 2e-3 * np.sqrt(K), f"max err {err}; first row got {D[0, :4]} want {ref[0, :4]}"
