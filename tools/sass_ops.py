"""Opcode histogram per kernel of the shipped library (evidence for which hardware paths the kernels use):
    python tools/sass_ops.py
Tensor-core / TMA / barrier mnemonics to look for: HMMA (mma.sync), HGMMA (wgmma), WARPGROUP (wgmma fences / waits),
UBLKCP (cp.async.bulk), SYNCS (mbarrier), LDGSTS (cp.async), BAR (named barriers), MUFU."""
import collections
import os
import re
import subprocess
import sys

LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "nv_wavenet_b200", "lib", "libwavenet_infer.so")
KEY = ("HMMA", "HGMMA", "WARPGROUP", "UBLKCP", "SYNCS", "LDGSTS", "BAR", "MUFU", "LDS", "STS", "LDG", "STG", "FFMA", "FADD", "FMUL", "HFMA2", "HMUL2", "DFMA")
out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
kern, hist = None, collections.OrderedDict()
for line in out.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
        full = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().replace("(anonymous namespace)::", "")
        kern = full[:full.rfind("(")] if "(" in full else full
        hist[kern] = collections.Counter()
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", line)
    if m and kern:
        hist[kern][m.group(1)] += 1
print(f"# cuobjdump -sass {os.path.relpath(LIB)}  (sm_90a)  -- instruction counts per kernel; columns: total, then the mnemonics of interest")
for k, c in hist.items():
    tot = sum(c.values())
    if tot < 50:
        continue
    print(f"{k[:110]}\n    total {tot}  " + "  ".join(f"{n} {c[n]}" for n in KEY if c[n]))
