"""Serving a queue of prompted utterances: continuous batching with prompts (NVWaveNet.infer_many(prompts=...)) against static batches
of infer(prompt=P).

    python tools/serve_prompt_bench.py --out DIR [--utterances 192] [--rounds 3] [--seed 1]

Workload: the C3 model (fp16, R64 / S256 / A256, 20 layers, max dilation 512, lively seeded weights), 64 slots, windows of 4 000
samples, and a seeded queue of `utterances` utterances: each has a prompt of P in {1 000, 4 000, 8 000} samples (random codes) and
then 4 000-12 000 samples to generate, conditioned on a slice of one random conditioning tensor.
  continuous  infer_many(prompts=..., slots=64, window=4000): a slot takes the next queued utterance at the first window boundary
              after its utterance ends; the prompted utterances starting at a boundary are scored together and primed into their slots.
  static      batches of 64 in arrival order among the utterances of one P, each one call of infer(prompt=P, window=4000) up to its
              longest utterance.
The arms alternate, `rounds` times; each figure is the median over the rounds, with its min and max.  Reported: useful samples/s
(generated samples, the prompts excluded, over the wall time), the GPU time infer_many spends scoring and priming prompts ("prime_s")
and per prompted utterance, and the sizes of the groups of prompts that start together.  A separate phase times scoring and priming
groups of g in {1, 2, 8, 64} prompts of 4 000 samples on the same engine, per utterance: the scorer's chunk is 16384 / 64 = 256
steps whatever g is, so small groups run small launches.  The card's name, power limit and SM clocks come from a read-only nvidia-smi
query in the same run, before and after.  Writes DIR/serve_prompt_bench.json and prints it.
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nv_wavenet_b200.nv_wavenet import plan_slots  # noqa: E402
from tools.serve_bench import A, L, R, card, network  # noqa: E402

SLOTS, WINDOW = 64, 4000
PROMPTS = (1000, 4000, 8000)
LO, HI = 4000, 12000


def static_batches(net, conds, prompts, seeds):
    """Batches of SLOTS in arrival order among the utterances of each prompt length, each through one infer(prompt=P) call."""
    outs, by_p = [None] * len(conds), {}
    for u, p in enumerate(prompts):
        by_p.setdefault(p.numel(), []).append(u)
    for P, us in by_p.items():
        for b0 in range(0, len(us), SLOTS):
            batch = us[b0:b0 + SLOTS]
            longest = max(conds[u].size(2) for u in batch)
            cond = torch.zeros((2 * R, len(batch), L, longest), dtype=torch.float32, device="cuda")
            for j, u in enumerate(batch):
                cond[:, j, :, :conds[u].size(2)].copy_(conds[u])
            y = net.infer(cond, 0, seed=seeds[batch[0]], fp16=True, window=WINDOW, prompt=torch.stack([prompts[u] for u in batch]))
            del cond
            for j, u in enumerate(batch):
                outs[u] = y[j, :conds[u].size(2)]
    torch.cuda.synchronize()
    return outs


def group_cost(net, base, g, P=4000, reps=5):
    """GPU ms per utterance of scoring and priming g prompts of P samples through the engine's store, as infer_many does."""
    eng = net._engine(SLOTS, WINDOW, True)
    codes = torch.randint(0, A, (g, P), device="cuda", dtype=torch.int32)
    lh = base[:, :, :P].permute(2, 1, 0).unsqueeze(2).expand(P, L, g, 2 * R).contiguous()
    times = []
    for k in range(reps + 1):
        eng.reset_history()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for first in range(0, P, WINDOW):
            m = min(WINDOW, P - first)
            eng.set_conditioning_slots(lh[first:first + m], list(range(g)), first)
            eng.score_stream(codes[:, first:first + m], first)
        eng.prime_slots_from_score(list(range(g)), list(range(g)))
        b.record()
        torch.cuda.synchronize()
        if k:
            times.append(a.elapsed_time(b) / g)
    return {"g": g, "P": P, "ms_per_utterance": statistics.median(times), "min": min(times), "max": max(times)}


def summary(v):
    return {"median": statistics.median(v), "min": min(v), "max": max(v)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", default=None, help="directory for serve_prompt_bench.json")
    ap.add_argument("--utterances", type=int, default=192)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    for k in ("NVWN_FP16_KERNEL", "NVWN_LAT_CLUSTER", "NVWN_LAT_MAX_B", "NVWN_TC_TILE", "NVWN_TC_NODUP", "NVWN_TC_FUSED"):
        os.environ.pop(k, None)

    rng = np.random.default_rng(args.seed)
    plens = [int(v) for v in rng.choice(PROMPTS, args.utterances)]
    gens = [int(v) for v in rng.integers(LO, HI + 1, args.utterances)]
    lengths = [p + n for p, n in zip(plens, gens)]
    offsets = [int(v) for v in rng.integers(0, HI + 1, args.utterances)]
    seeds = [int(v) for v in rng.integers(0, 2 ** 62, args.utterances)]
    g = torch.Generator(device="cuda").manual_seed(args.seed)
    base = 0.5 * torch.randn((2 * R, L, 2 * HI + max(PROMPTS) + 1), generator=g, device="cuda")
    conds = [base[:, :, o:o + n] for o, n in zip(offsets, lengths)]
    prompts = [torch.randint(0, A, (p,), generator=g, device="cuda", dtype=torch.int32) for p in plens]
    net = network(args.seed)
    info = card()

    plan = plan_slots(gens, SLOTS, WINDOW)
    groups = {}
    for _, t in plan:
        groups[t] = groups.get(t, 0) + 1
    useful = sum(gens)

    # warm-up of both arms: engine creation, weight upload, the scorer's scratch and first launches
    net.infer_many([c[:, :, :2 * WINDOW] for c in conds[:SLOTS]], seeds[:SLOTS], slots=SLOTS, window=WINDOW, fp16=True,
                   prompts=[torch.zeros(WINDOW, dtype=torch.int32, device="cuda") + 128] * SLOTS)
    static_batches(net, [c[:, :, :2 * WINDOW] for c in conds[:SLOTS]], [torch.full((1000,), 128, dtype=torch.int32, device="cuda")] * SLOTS,
                   seeds[:SLOTS])

    cont_t, stat_t, prime_s, gen_s = [], [], [], []
    same = True
    for _ in range(args.rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        timing = {}
        cont = net.infer_many(conds, seeds, slots=SLOTS, window=WINDOW, fp16=True, timing=timing, prompts=prompts)
        cont_t.append(time.perf_counter() - t0)
        prime_s.append(timing["prime_s"])
        gen_s.append(timing["generate_s"])
        t0 = time.perf_counter()
        stat = static_batches(net, conds, prompts, seeds)
        stat_t.append(time.perf_counter() - t0)
        same = same and all(torch.equal(a[:p.numel()], b[:p.numel()]) for a, b, p in zip(cont, stat, prompts))
        del cont, stat
    costs = [group_cost(net, base, g) for g in (1, 2, 8, 64)]
    after = card()
    launch = net._engine(SLOTS, WINDOW, True).launch_info()

    res = {
        "workload": {"model": "C3", "dtype": "fp16", "slots": SLOTS, "window": WINDOW, "utterances": args.utterances, "prompts": list(PROMPTS),
                     "generated": [LO, HI], "seed": args.seed, "rounds": args.rounds, "useful_samples": useful,
                     "prompt_samples": sum(plens)},
        "card": info, "card_after": after, "launch": {k: launch[k] for k in ("kernel", "grid", "batch_per_cta", "cluster")},
        "continuous": {"seconds": summary(cont_t), "useful_samples_per_s": summary([useful / t for t in cont_t]),
                       "prime_s": summary(prime_s), "generate_s": summary(gen_s),
                       "prime_ms_per_prompted_utterance": summary([1e3 * s / args.utterances for s in prime_s]),
                       "prompt_groups": sorted(groups.values(), reverse=True)},
        "static": {"seconds": summary(stat_t), "useful_samples_per_s": summary([useful / t for t in stat_t])},
        "speedup": statistics.median(stat_t) / statistics.median(cont_t),
        "prompts_returned_as_given": same,
        "score_prime_by_group": costs,
    }
    line = json.dumps(res)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "serve_prompt_bench.json"), "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
