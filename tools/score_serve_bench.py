"""Scoring a queue of utterances of different lengths: packed scoring (NVWaveNet.log_likelihood_many) against static padded batches
(NVWaveNet.log_likelihood), and what the packed kernels' masks cost.

    python tools/score_serve_bench.py --out DIR [--utterances 512] [--seed 2026] [--rounds 2]

C3 model (R64 / S256 / A256, 20 layers, max dilation 512, fp16) with seeded weights, 64 rows, a queue of 512 utterances with lengths
uniform in [8 000, 48 000] (seed 2026) and seeded audio.  Utterance u in arrival order has the conditioning pool[:, :, o_u : o_u + n_u]
of one seeded pool, o_u = 512 * (u mod 64), so both arms score every utterance on the same conditioning and audio.  For W = 4 096 and
W = 16 000, after one warm-up pass of each arm (which also checks that both give every utterance the same bits), `rounds` rounds
alternate the arms, each pass timed with CUDA events and ending in a device synchronise:
  static  groups of 64 in arrival order, each padded to its longest utterance (code 128 after an utterance's end), one
          log_likelihood(cond, audio, window=W) per group;
  packed  log_likelihood_many(conds, audios, slots=64, window=W).
Reported per arm: medians of time, useful samples/s (the real samples), scored samples/s (rows x samples the scorer ran) and the
packed / static ratios.  Mask cost: 64 x 16 000 samples in one engine of 16 000 samples with a start only at sample 0,
score_stream_packed against score_stream (device audio, flags and outputs), alternated over 10 calls each after a warm-up, CUDA
events; both give the same bits.  The card's name, power limit and max SM clock come from the read-only nvidia-smi query of
tools/score_bench.py, in the same run.  Writes DIR/score_serve_bench.json and prints it as one line.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nv_wavenet_b200.nv_wavenet import _packed_windows, plan_packed  # noqa: E402
from tools.score_bench import card  # noqa: E402
from tools.score_stream_bench import A, L, MD, R, S, c3_net, timed_call  # noqa: E402

SLOTS, LO, HI, SHIFT = 64, 8000, 48000, 512
MASK_SAMPLES = 16000


def static(net, conds_pool, audios, lengths, window):
    """Groups of SLOTS in arrival order, each padded to its longest, through log_likelihood(window=W): per utterance its logp."""
    outs = []
    for g0 in range(0, len(lengths), SLOTS):
        group = list(range(g0, min(g0 + SLOTS, len(lengths))))
        n = max(lengths[u] for u in group)
        # row j's conditioning is pool[:, :, 512 j : 512 j + n], a strided view the call materializes a window at a time
        p = conds_pool
        cond = p.as_strided((p.size(0), len(group), p.size(1), n), (p.stride(0), SHIFT * p.stride(2), p.stride(1), p.stride(2)))
        audio = torch.full((len(group), n), 128, dtype=torch.int32, device="cuda")
        for j, u in enumerate(group):
            audio[j, :lengths[u]] = audios[u]
        lp = net.log_likelihood(cond, audio, window=window)
        outs += [lp[j, :lengths[u]] for j, u in enumerate(group)]
    return outs


def mask_cost(net, g, calls=10):
    """score_stream_packed with a start only at 0 against score_stream, 64 x MASK_SAMPLES in one engine: ms per call of each."""
    eng = net._engine(SLOTS, MASK_SAMPLES, True)
    eng.set_conditioning(0.5 * torch.randn((MASK_SAMPLES, L, SLOTS, 2 * R), generator=g, device="cuda"), 0, MASK_SAMPLES)
    audio = torch.randint(0, A, (SLOTS, MASK_SAMPLES), generator=g, device="cuda", dtype=torch.int32)
    starts = torch.zeros((SLOTS, MASK_SAMPLES), dtype=torch.uint8, device="cuda")
    starts[:, 0] = 1
    plain = lambda: eng.score_stream(audio, 0)
    packed = lambda: eng.score_stream_packed(audio, starts, 0)
    a, b = plain(), packed()
    torch.cuda.synchronize()
    equal = torch.equal(a.view(torch.int32), b.view(torch.int32))
    ms = {"plain": [], "packed": []}
    for _ in range(calls):
        ms["plain"].append(timed_call(plain)[1])
        ms["packed"].append(timed_call(packed)[1])
    med = {k: float(np.median(v)) for k, v in ms.items()}
    return {"rows": SLOTS, "samples": MASK_SAMPLES, "calls": calls, "score_stream_ms": ms["plain"], "score_stream_packed_ms": ms["packed"],
            "score_stream_ms_median": med["plain"], "score_stream_packed_ms_median": med["packed"],
            "packed_over_plain": med["packed"] / med["plain"], "bit_equal": bool(equal)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--utterances", type=int, default=512)
    ap.add_argument("--seed", type=int, default=2026)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("score_serve_bench needs a CUDA device")
    rng = np.random.default_rng(args.seed)
    lengths = [int(v) for v in rng.integers(LO, HI + 1, args.utterances)]
    g = torch.Generator(device="cuda").manual_seed(args.seed)
    pool = 0.5 * torch.randn((2 * R, L, SHIFT * (SLOTS - 1) + HI), generator=g, device="cuda")
    conds = [pool[:, :, SHIFT * (u % SLOTS):SHIFT * (u % SLOTS) + n] for u, n in enumerate(lengths)]
    audios = [torch.randint(0, A, (n,), generator=g, device="cuda", dtype=torch.int32) for n in lengths]
    net = c3_net(args.seed)
    info = card()

    useful = sum(lengths)
    static_scored = sum(SLOTS * max(lengths[b:b + SLOTS]) for b in range(0, len(lengths), SLOTS))
    plan = plan_packed(lengths, SLOTS)
    res = {"card": info, "model": {"R": R, "S": S, "A": A, "L": L, "max_dilation": MD, "dtype": "fp16"},
           "queue": {"utterances": len(lengths), "lengths": [LO, HI], "seed": args.seed, "rows": SLOTS, "useful_samples": useful},
           "rounds": args.rounds, "windows": {}}
    for W in (4096, 16000):
        packed_scored = SLOTS * sum(n for _, n, _ in _packed_windows(plan, lengths, W))
        run_static = lambda: static(net, pool, audios, lengths, W)
        split = {}
        run_packed = lambda: net.log_likelihood_many(conds, audios, slots=SLOTS, window=W, timing=split)
        ref, got = run_static(), run_packed()
        equal = all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(ref, got))
        del ref, got
        ms = {"static": [], "packed": []}
        produce, score = [], []
        for _ in range(args.rounds):
            ms["static"].append(timed_call(run_static)[1])
            ms["packed"].append(timed_call(run_packed)[1])
            produce.append(split["produce_s"] * 1e3)
            score.append(split["score_s"] * 1e3)
        med = {k: float(np.median(v)) for k, v in ms.items()}
        arm = lambda k, scored: {"ms": ms[k], "ms_median": med[k], "scored_samples": scored, "real_fraction": useful / scored,
                                 "useful_samples_per_s": useful / (med[k] * 1e-3), "scored_samples_per_s": scored / (med[k] * 1e-3)}
        res["windows"][str(W)] = {
            "static": arm("static", static_scored), "packed": arm("packed", packed_scored),
            "packed_fill_ms_median": float(np.median(produce)), "packed_score_ms_median": float(np.median(score)),
            "useful_rate_ratio": med["static"] / med["packed"],
            "cost_per_scored_sample_ratio": (med["packed"] / packed_scored) / (med["static"] / static_scored),
            "bit_equal": bool(equal)}
        torch.cuda.empty_cache()
    res["mask_cost"] = mask_cost(net, g)
    res["card_after"] = card()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "score_serve_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
