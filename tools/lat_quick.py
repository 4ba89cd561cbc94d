"""Quick timing of the fp16 kernels at the C3 model (kernel-only, CUDA events): python tools/lat_quick.py [B ...]"""
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, ".")
import nv_wavenet_b200 as nw
from tests import refgen

L, R, S, A, md = 20, 64, int(os.environ.get("S", 256)), 256, 512
N = int(os.environ.get("N", 4000))
Bs = [int(a) for a in sys.argv[1:]] or [64]
from nv_wavenet_b200 import _lib
print(json.dumps({"three_cta_clusters_resident_at_once": {f"{rows}_rows": _lib.lib().nvwn_debug_lat_max_clusters(S, rows) for rows in (8, 16)}}))
for B in Bs:
    w = refgen.lively_inputs(3, R, S, A, L, min(B, 16), 8)
    rng = np.random.default_rng(0)
    for kern in os.environ.get("KERNELS", "lat,tc").split(","):
        os.environ["NVWN_FP16_KERNEL"] = kern
        e = nw.NVWavenetInfer(L, md, B, N, R=R, S=S, A=A, dtype=nw.FP16)
        e.load(w)
        # conditioning: small random, generated on the device chunk by chunk
        per = L * B * 2 * R
        chunk = max(1, (64 << 20) // per)
        g = torch.Generator(device="cuda"); g.manual_seed(1)
        for s0 in range(0, N, chunk):
            m = min(chunk, N - s0)
            lh = (torch.rand((m, L, B, 2 * R), device="cuda", generator=g) - 0.5) * 0.5
            e.set_conditioning(lh, s0, m)
        torch.cuda.synchronize()
        e.set_selectors(torch.rand((N, B), device="cuda", generator=g))
        e.reset_history()
        y = torch.zeros((B, N), dtype=torch.int32, device="cuda")
        e.run(min(N, 200), B, None); torch.cuda.synchronize()
        e.reset_history()
        t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
        t0.record(); e.run(N, B, y); t1.record(); torch.cuda.synchronize()
        ms = t0.elapsed_time(t1)
        yy = y.cpu().numpy()
        print(json.dumps({"kernel": kern, "B": B, "S": S, "N": N, "ms": round(ms, 3), "khz_per_utt": round(N / ms, 2), "Msamples_s": round(B * N / ms / 1e3, 3),
                          "cycles_per_sample": round(ms * 1e-3 * 1.965e9 / N), "uniq": int(len(np.unique(yy))), "info": e.launch_info()}), flush=True)
        e.close()
