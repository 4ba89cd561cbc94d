"""Teacher-forced scoring throughput (nvwn_score) against forced generation of the same audio on the same engine.

    python tools/score_bench.py --out DIR [--calls 5] [--warmup 1] [--workloads c3,r128]

Workloads (fp16, lively seeded weights, random conditioning and audio):
  c3    R64 / S256 / A256, 20 layers, max dilation 512, 64 utterances x 16 000 samples
  r128  R128 / S256 / A256, 30 layers, max dilation 512, 16 utterances x 16 000 samples
Each is timed with CUDA events over `calls` calls after `warmup` calls.  Reported: ms per call, samples/s, TFLOP/s counted as
2 x weights x samples, and the two lower bounds of the design as built (DESIGN.md §5.4): the dense fp16 tensor-core peak and the
HBM bytes its buffers move.  The card's name, power limit and max SM clock come from a read-only nvidia-smi query.
Writes DIR/score_bench.json and prints it.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nv_wavenet_b200 as nw  # noqa: E402
from tests import refgen  # noqa: E402

WORKLOADS = {"c3": (64, 256, 256, 20, 512, 64, 16000), "r128": (128, 256, 256, 30, 512, 16, 16000)}
PEAK_FP16_TFLOPS = 989.4          # H100 SXM5 data sheet, dense fp16 tensor core
PEAK_HBM_TBS = 3.35               # H100 SXM5 80 GB data sheet


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as ex:                                     # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(0), "query_error": str(ex)}


def weights_per_sample(R, S, A, L):
    """Multiply-adds per sample: the matrices every generation step multiplies by."""
    return L * (2 * R * 2 * R + R * R + S * R) + A * S + A * A


def bytes_per_sample(R, S, A, L):
    """HBM bytes per (t, b) row of the scorer's buffers (DESIGN.md §5.4): conditioning readback (fp16 store in, fp32 out, fp32
    back in by the layers), embedding, per layer [x | x(t-d)] fp16 in, fp32 residual in + out, fp16 x and h out, H back in for
    the skip GEMM, logp out.  Weight traffic (once per CTA per launch) is left out."""
    lh = L * 2 * R * (2 + 4 + 4)
    embed = 4 * R + 2 * R
    layers = L * (2 * 2 * R + 4 * R + 4 * R + 2 * R + 2 * R)
    return lh + embed + layers + 2 * L * R + 4


def timed(fn, calls, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(calls + 1)]
    ms = []
    ev[0].record()
    for i in range(calls):
        fn()
        ev[i + 1].record()
    torch.cuda.synchronize()
    for i in range(calls):
        ms.append(ev[i].elapsed_time(ev[i + 1]))
    return ms


def run(name, calls, warmup):
    R, S, A, L, md, B, N = WORKLOADS[name]
    w = refgen.lively_inputs(17, R, S, A, L, 1, 1)
    e = nw.NVWavenetInfer(L, md, B, N, R=R, S=S, A=A, dtype=nw.FP16)
    e.load(w)
    g = torch.Generator(device="cuda").manual_seed(18)
    for first in range(0, N, 1000):                             # random conditioning, uploaded in chunks of samples
        n = min(1000, N - first)
        e.set_conditioning(0.5 * torch.randn((n, L, B, 2 * R), generator=g, device="cuda"), first, n)
    audio = torch.randint(0, A, (B, N), generator=g, device="cuda", dtype=torch.int32)
    logp = [None]

    def score():
        logp[0] = e.score(audio)
    y = torch.empty((B, N), dtype=torch.int32, device="cuda")
    e.set_forced(audio)

    def generate():
        e.run(N, B, y)
    ms_score = timed(score, calls, warmup)
    ms_gen = timed(generate, calls, warmup)
    samples = B * N
    t = float(np.median(ms_score)) * 1e-3
    flops = 2.0 * weights_per_sample(R, S, A, L) * samples
    nbytes = float(bytes_per_sample(R, S, A, L)) * samples
    t_flop, t_byte = flops / (PEAK_FP16_TFLOPS * 1e12), nbytes / (PEAK_HBM_TBS * 1e12)
    tg = float(np.median(ms_gen)) * 1e-3
    return {
        "workload": name, "R": R, "S": S, "A": A, "L": L, "max_dilation": md, "batch": B, "samples": N,
        "score_ms": ms_score, "score_ms_median": t * 1e3, "score_samples_per_s": samples / t, "score_tflops": flops / t / 1e12,
        "flop_bound_ms": t_flop * 1e3, "byte_bound_ms": t_byte * 1e3, "bytes_per_sample": bytes_per_sample(R, S, A, L),
        "nearer_bound": "flop" if t_flop > t_byte else "bytes", "fraction_of_nearer_bound": max(t_flop, t_byte) / t,
        "generate_ms": ms_gen, "generate_ms_median": tg * 1e3, "generate_samples_per_s": samples / tg,
        "generate_kernel": e.launch_info()["kernel"], "speedup_vs_forced_generation": tg / t,
        "mean_neg_logp": float(-logp[0].double().mean().item()),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--workloads", default="c3,r128")
    a = ap.parse_args()
    res = {"card": card(), "results": [run(n, max(a.calls, 5), a.warmup) for n in a.workloads.split(",")]}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "score_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
