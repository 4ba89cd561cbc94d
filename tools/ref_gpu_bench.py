"""GPU baseline: the reference's own kernels (oracle/_ref/ref_gpu_harness, unmodified nv_wavenet.cuh rebuilt for
sm_90a) timed exactly like nv_wavenet_perf.cu:67-87 (run_chunks incl. chunked D2H), next to our kernels, same inputs."""
import json
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
import nv_wavenet_b200 as nw
from oracle import ref_gpu
from tests import refgen

R, S, A, L, MD = 64, 256, 256, 20, 512
out = {}
for prec, B, N in ((16, 64, 2000), (16, 8, 2000), (32, 64, 1000), (32, 16, 1000)):
    w = refgen.synthetic_inputs(1, R, S, A, L, B, N)          # reference-test scale: no saturation in the fp16-accumulating reference
    row = {}
    for mode, name in ((3, "persistent"), (2, "dual_block"), (1, "single_block")):
        try:
            r = ref_gpu.run(w, prec, R, S, A, L, MD, B, N, mode=mode, chunk=2048, reps=2)
            row["reference_" + name] = {"khz_per_utterance": r["khz"], "samples_per_s": r["samples_per_s"]}
        except Exception as ex:          # noqa: BLE001
            row["reference_" + name] = {"error": str(ex)[:200]}
    e = nw.NVWavenetInfer(L, MD, B, N, R=R, S=S, A=A, dtype=nw.FP16 if prec == 16 else nw.FP32)
    e.load(w); e.set_inputs(w["Lh"], w["selectors"])
    y = torch.zeros((B, N), dtype=torch.int32).pin_memory()
    for it in range(3):
        e.reset_history()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        e.run_chunks(2048, lambda *a: None, N, B, y)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
    row["ours"] = {"khz_per_utterance": N / ms, "samples_per_s": N * B / (ms * 1e-3), "kernel": e.launch_info()["kernel"]}
    out[f"fp{prec}_B{B}"] = row
    print(f"fp{prec} B={B}", json.dumps(row), flush=True)
json.dump(out, open("gpurun_out/ref_gpu_baseline.json", "w"), indent=1)
