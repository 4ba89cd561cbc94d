"""Debug tool: clock64 timeline of one sample of the latency-mode kernel (block 0; compute thread 0 and the producer lane).
python tools/lat_trace.py [B] [sample]"""
import ctypes as C
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
import os
os.environ.setdefault("NVWN_FP16_KERNEL", "lat")
# NVWN_LAT_CLUSTER=0 traces the single-CTA kernel; default: the cluster kernel (role 0 = chain CTA, role 1 = tail CTA, role 2 = prep CTA:
# thread 0 of each, the prep only around its half of the output layers)
import nv_wavenet_b200 as nw
from nv_wavenet_b200 import _lib
from tests import refgen

L, R, S, A, md = 20, 64, int(os.environ.get("S", 256)), 256, 512
B = int(sys.argv[1]) if len(sys.argv) > 1 else 64
T = int(sys.argv[2]) if len(sys.argv) > 2 else 30
N = T + 10
w = refgen.lively_inputs(3, R, S, A, L, B, N)
e = nw.NVWavenetInfer(L, md, B, N, R=R, S=S, A=A, dtype=nw.FP16)
e.load(w); e.set_inputs(w["Lh"], w["selectors"])
lib = _lib.lib()
lib.nvwn_debug_trace.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
assert lib.nvwn_debug_trace(e._h, T, None, 0) == 0
e.run(N, B, None); torch.cuda.synchronize()
buf = np.zeros(3 * 1024, np.uint64)
assert lib.nvwn_debug_trace(e._h, T, buf.ctypes.data, 1) == 0
names = {1: "sample start (ys read)", 2: "x0 built", 10: "h exchanged", 11: "layer done (x exchanged)", 12: "cur+prev GEMM issued", 13: "probes issued",
         14: "res done", 15: "skip issued", 16: "tail: h seen", 17: "tail: prev part starts", 18: "tail: pre-activation shipped", 20: "relu(skip) sent", 21: "relu(Zs) exchanged",
         22: "logits half received", 23: "sample done", 24: "Zs done", 30: "prep: output half starts", 33: "prep: logits half sent"}
ev = []
for role in range(3):
    for v in buf[role * 1024:(role + 1) * 1024]:
        v = int(v)
        if v:
            ev.append((v & 0xFFFFFFFFFFFF, role, v >> 48))
ev.sort()
t0 = ev[0][0]
prev = {0: t0, 1: t0, 2: t0}
for clk, role, tag in ev:
    nm = names.get(tag, ("prod: layer %d issued" % (tag - 100)) if 100 <= tag < 200 else ("prod: out load %d issued" % (tag - 200)) if tag >= 200 else str(tag))
    print(f"{clk - t0:8d} (+{clk - prev[role]:6d})  role{role}  {nm}")
    prev[role] = clk
print("total cycles in sample:", ev[-1][0] - t0, "events", len(ev))
