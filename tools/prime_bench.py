"""Prompted generation: the prompt run by forced generation against the scorer and a prime (nvwn_prime_from_score), then free
generation in both.

    python tools/prime_bench.py --out DIR [--calls 5] [--warmup 1]

Two workloads with lively seeded weights (the scales of tests/refgen.py lively_inputs), seeded conditioning (a seeded block of 1 000
samples, repeated) and a seeded prompt, each on one fp16 engine of the whole length:
  c3    C3 model (R64 / S256 / A256, 20 layers, max dilation 512), 64 utterances x (16 000-sample prompt + 16 000 generated);
  r128  R128 / S256 / A256, 30 layers, max dilation 512, 16 utterances x (16 000 + 4 000).
Two arms on the same engine, inputs and selectors (device Philox, one seed), alternated call by call after `warmup` rounds:
  a  forced generation of the prompt (nvwn_set_forced, nvwn_run_stream over [0, P)), then free generation;
  b  nvwn_score_stream over [0, P), nvwn_prime_from_score, then free generation.
Each call is timed with CUDA events: the prompt stage plus the first generated sample (time to the first sample), and the whole call.
The first generated sample runs as a launch of its own with dumps in both arms, so the run also checks that b's logits of step P are
within the fp16 rule (1e-2 of max(|z|, 0.25 max|z| of the utterance)) of a's.  The card's name, power limit and max SM clock come from
the read-only nvidia-smi query of tools/score_bench.py.  Writes DIR/prime_bench.json and prints it.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import nv_wavenet_b200 as nw  # noqa: E402
from tests import refgen  # noqa: E402
from tools.score_bench import card  # noqa: E402

WORKLOADS = {
    "c3": dict(R=64, S=256, L=20, B=64, P=16000, G=16000),
    "r128": dict(R=128, S=256, L=30, B=16, P=16000, G=4000),
}
A, MD, BLOCK = 256, 512, 1000


def setup(R, S, L, B, P, G, seed):
    N = P + G
    w = refgen.lively_inputs(seed, R, S, A, L, 1, 1)
    e = nw.NVWavenetInfer(L, MD, B, N, nw.AUTO, True, R=R, S=S, A=A, dtype=nw.FP16)
    e.load(w)
    g = torch.Generator(device="cuda").manual_seed(seed)
    lh = 0.5 * torch.randn((BLOCK, L, B, 2 * R), generator=g, device="cuda")
    for k in range(0, N, BLOCK):
        e.set_conditioning(lh[:min(BLOCK, N - k)], k, min(BLOCK, N - k))
    e.set_selectors_random(seed)
    forced = torch.randint(0, A, (B, N), generator=g, device="cuda", dtype=torch.int32)
    return e, forced


def call(e, forced, arm, B, P, G):
    """One prompted generation; returns (ms to the first generated sample, ms in all, logits of step P [B][A])."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    e.reset_history()
    ev[0].record()
    if arm == "a":
        e.set_forced(forced)
        e.run_stream(0, P, B)
        e.set_forced(None)
    else:
        e.score_stream(forced[:, :P], 0)
        e.prime_from_score()
    e.run_stream(P, 1, B, dump_activations=True)
    ev[1].record()
    e.run_stream(P + 1, G - 1, B)
    ev[2].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]), ev[0].elapsed_time(ev[2]), e.get_za()


def fp16_rule(ref, got):
    scale = np.abs(ref).max(axis=-1, keepdims=True)
    err = np.abs(got - ref)
    return bool(np.all(err <= 1e-2 * np.maximum(np.abs(ref), 0.25 * scale))), float((err / scale).max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prime_bench needs a CUDA device")
    calls = max(a.calls, 5)
    res = {"card": card(), "calls": calls, "warmup": a.warmup, "max_dilation": MD, "A": A, "dtype": "fp16"}
    for name, wl in WORKLOADS.items():
        B, P, G = wl["B"], wl["P"], wl["G"]
        e, forced = setup(wl["R"], wl["S"], wl["L"], B, P, G, 51)
        for _ in range(a.warmup):
            call(e, forced, "a", B, P, G); call(e, forced, "b", B, P, G)
        ms = {arm: {"first": [], "total": []} for arm in "ab"}
        ok, worst = True, 0.0
        for _ in range(calls):
            za = {}
            for arm in "ab":
                first, total, za[arm] = call(e, forced, arm, B, P, G)
                ms[arm]["first"].append(first)
                ms[arm]["total"].append(total)
            good, err = fp16_rule(za["a"], za["b"])
            ok, worst = ok and good, max(worst, err)
        med = {arm: {k: float(np.median(v)) for k, v in ms[arm].items()} for arm in "ab"}
        res[name] = dict(wl, kernel=e.launch_info()["kernel"],
                         forced_ms=ms["a"], primed_ms=ms["b"],
                         forced_first_ms_median=med["a"]["first"], forced_total_ms_median=med["a"]["total"],
                         primed_first_ms_median=med["b"]["first"], primed_total_ms_median=med["b"]["total"],
                         first_sample_speedup=med["a"]["first"] / med["b"]["first"],
                         total_speedup=med["a"]["total"] / med["b"]["total"],
                         primed_prompt_samples_per_s=B * P / (med["b"]["first"] * 1e-3),
                         step_P_logits_within_fp16_rule=ok, step_P_max_err_over_scale=worst)
        e.close()
        del e, forced
        torch.cuda.empty_cache()
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "prime_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
