"""Generates tests/golden/reference_gpu.npz with the reference's OWN CUDA kernels (oracle/_ref/ref_gpu_harness: the
unmodified nv_wavenet.cuh PERSISTENT kernel, built by `make -C oracle refgpu`) on the two cases of
tests/test_gpu_vs_reference_gpu.py.  Needs a GPU and the built harness; the test only reads the committed .npz.

    python tests/golden/make_golden_refgpu.py

Stores, per case, the sampled indices `y` [B][N] and the last sample's logits `za` [B][A].  Inputs are not stored:
tests/refgen.py regenerates them.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_gpu                          # noqa: E402
from tests import test_gpu_vs_reference_gpu as t    # noqa: E402


def main():
    out = {}
    for name, (w, prec, B, N, chunk) in t.cases().items():
        ref = ref_gpu.run(w, prec, t.R, t.S, t.A, t.L, t.MD, B, N, mode=3, chunk=chunk)
        out[f"{name}/y"] = ref["y"]
        out[f"{name}/za"] = ref["za"]
        print(name, ref["y"].shape, float(np.abs(ref["za"]).max()))
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_gpu.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
