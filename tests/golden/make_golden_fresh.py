"""Generates tests/golden/reference_cpu_fresh.npz: the reference's OWN CPU model (oracle/_ref/libnvwn_ref.so, the
unmodified nv_wavenet_reference.cpp built by oracle/Makefile) on the fresh shapes of
tests/test_oracle_pin.py::test_oracle_vs_reference_cpu_fresh_shapes.  The test only reads the committed .npz.

    python tests/golden/make_golden_fresh.py

Stores, per case and run, the sampled indices and the last sample's activations (Xt, skip, Zs, Za, p).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import pyoracle as po          # noqa: E402
from tests import test_oracle_pin as t     # noqa: E402


def main():
    po.build()
    if not po.have_ref():
        raise SystemExit("oracle/_ref/libnvwn_ref.so is missing: build it with `make -C oracle ref REF=<reference checkout>`")
    out = {}
    for shape in t.FRESH_SHAPES:
        for gen in ("uniform", "lively"):
            R, S, A, L, B, bs, N, md = shape
            w = t.fresh_inputs(shape, gen)
            ref = po.RefCPU(L, B, N, R, S, A, md); ref.load(w); ref.set_inputs(w["Lh"], w["selectors"])
            key = t.fresh_key(shape, gen)
            for it in range(t.FRESH_ITERS):
                out[f"{key}/{it}/y"] = ref.run(N, bs)
                for k, v in ref.activations().items():
                    out[f"{key}/{it}/{k}"] = v
            print(key, "ok")
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_cpu_fresh.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
