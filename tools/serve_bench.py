"""Serving a queue of utterances of different lengths: continuous batching (NVWaveNet.infer_many), continuous batching from mel
frames (NVWaveNet.infer_many_from_features) and static batches.

    python tools/serve_bench.py --out DIR [--utterances 256] [--seed 1]

Workload: the C3 model (fp16, R64 / S256 / A256, 20 layers, max dilation 512, lively seeded weights), 64 slots, windows of
4 000 samples, and a seeded mix of `utterances` utterances of whole frames of 200 samples, uniform in [16 000, 160 000] samples.
The first and third arms condition each utterance on a slice of one random conditioning tensor; the second on its own random
mel frames (80 channels) through a seeded conditioning network of the reference's geometry (upsampling window 800, stride 200).
  continuous  infer_many(slots=64, window=4000): a slot takes the next queued utterance at the first window boundary after its
              utterance ends.
  mel         infer_many_from_features(slots=64, window=4000): the same schedule; each window's conditioning is produced on the
              device from the frames, on a side stream one window ahead of generation.
  static      batches of 64 in arrival order, each generated up to its longest utterance by the loop of infer(window=4000)
              (per window: conditioning of the whole batch, selectors, run_stream, yOut).  The loop is run here with the window's
              conditioning assembled from the same slices, because infer() wants the batch's whole conditioning tensor at once
              (64 x 160 000 samples x 20 x 128 fp32 = 105 GB).
Reported: useful samples/s of each arm (the sum of the lengths over the wall time), the padding fraction of the static batches
(computed from the lengths), the idle slot fraction of the continuous run, the GPU time infer_many spends in restarts and
per-slot uploads, the mel arm's production time per window and the time generation waited for it (zero when production is
hidden), and the bytes each arm's queued inputs would take (from shapes: fp32 conditioning [2R][L][n] against frames [80][T]).
A separate phase then times the production of one window of 64 slots alone, and splits it by kernel (upsampling, projection,
masking, store conversion) under torch.profiler.  The card's name, power limit and SM clock come from a read-only nvidia-smi query in the same run.
Writes DIR/serve_bench.json and prints it.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nv_wavenet_b200.nv_wavenet import NVWaveNet, plan_slots  # noqa: E402
from tests import refgen  # noqa: E402

R, S, A, L, MD = 64, 256, 256, 20, 512
SLOTS, WINDOW = 64, 4000
LO, HI = 16000, 160000
MEL, UP_WINDOW, STRIDE = 80, 800, 200


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock, max_clock = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power, "sm_clock": clock, "max_sm_clock": max_clock}
    except Exception as ex:                                     # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(0), "query_error": str(ex)}


def network(seed):
    """NVWaveNet of the C3 shape with lively random weights (tests/refgen.py), through its public constructor."""
    w = refgen.lively_inputs(seed, R, S, A, L, 1, 1)
    tt = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to("cuda")
    cm = lambda flat, M, K: np.ascontiguousarray(flat.reshape(K, M).T)
    dilate = [tt(np.stack([cm(w["Wprev"][l], 2 * R, R), cm(w["Wcur"][l], 2 * R, R)], axis=2)) for l in range(L)]
    return NVWaveNet(embedding_prev=tt(w["embPrev"]), embedding_curr=tt(w["embCur"]),
                     conv_out_weight=tt(cm(w["Wzs"], A, S)[:, :, None]), conv_end_weight=tt(cm(w["Wza"], A, A)[:, :, None]),
                     dilate_weights=dilate, dilate_biases=[tt(w["Bh"][l]) for l in range(L)], max_dilation=MD,
                     res_weights=[tt(cm(w["Wres"][l], R, R)[:, :, None]) for l in range(L - 1)],
                     res_biases=[tt(w["Bres"][l]) for l in range(L - 1)],
                     skip_weights=[tt(cm(w["Wskip"][l], S, R)[:, :, None]) for l in range(L)],
                     skip_biases=[tt(w["Bskip"][l]) for l in range(L)], use_embed_tanh=True)


def conditioning_network(seed):
    """Seeded upsampling ConvTranspose1d(80, 80, 800, stride 200) and 1x1 projection to L * 2R, scaled so that the conditioning
    has a standard deviation of about 0.5 like the slices of the other arms."""
    rng = np.random.default_rng(seed + 1)
    taps = UP_WINDOW // STRIDE
    return ((rng.standard_normal((MEL, MEL, UP_WINDOW)) / np.sqrt(MEL * taps)).astype(np.float32),
            (0.1 * rng.standard_normal(MEL)).astype(np.float32),
            (0.5 * rng.standard_normal((L * 2 * R, MEL)) / np.sqrt(MEL)).astype(np.float32),
            (0.1 * rng.standard_normal(L * 2 * R)).astype(np.float32))


def production_split(net, mels, cnet, reps=5):
    """Production of one window for all SLOTS slots, without generation: event time per window, then its kernels' device time
    per window under torch.profiler (a run of its own), grouped as upsampling, projection, masking and store conversion."""
    eng = net._engine(SLOTS, 2 * WINDOW, True)
    eng.reset_history()
    eng.cond_producer_set_weights(*cnet, STRIDE)
    eng.cond_producer_set_slots(range(SLOTS), mels[:SLOTS], [0] * SLOTS)
    eng.cond_producer_run_slots(range(SLOTS), 0, WINDOW)               # warm-up
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for k in range(reps):
        eng.cond_producer_run_slots(range(SLOTS), k * WINDOW, WINDOW)
    b.record()
    torch.cuda.synchronize()
    out = {"ms_per_window": a.elapsed_time(b) / reps}
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(reps):
            eng.cond_producer_run_slots(range(SLOTS), k * WINDOW, WINDOW)
        torch.cuda.synchronize()
    groups = {"upsample": 0.0, "project": 0.0, "mask": 0.0, "convert": 0.0, "other": 0.0}
    for item in prof.key_averages():
        us = getattr(item, "self_device_time_total", None)
        if us is None:
            us = item.self_cuda_time_total
        name = item.key
        g = ("upsample" if "upsample_slots" in name else "project" if "project" in name else "mask" if "mask_slots" in name
             else "convert" if "convert_rows" in name or "cond_rows" in name else "other")
        groups[g] += us / 1e3 / reps
    out["kernel_ms_per_window"] = groups
    out["kernels"] = sorted({item.key for item in prof.key_averages()})
    return out


def static_batches(net, conds, seeds):
    """Batches of SLOTS in arrival order through the loop of infer(window=WINDOW); returns the per-utterance outputs."""
    eng = net._engine(SLOTS, WINDOW, True)
    outs = [torch.empty(c.size(2), dtype=torch.int32, device="cuda") for c in conds]
    stage = torch.empty((SLOTS, WINDOW), dtype=torch.int32, device="cuda")
    for b0 in range(0, len(conds), SLOTS):
        batch = list(range(b0, min(b0 + SLOTS, len(conds))))
        longest = max(conds[u].size(2) for u in batch)
        eng.reset_history()
        for first in range(0, longest, WINDOW):
            n = min(WINDOW, longest - first)
            lh = torch.zeros((n, L, SLOTS, 2 * R), dtype=torch.float32, device="cuda")
            for j, u in enumerate(batch):
                m = min(n, conds[u].size(2) - first)
                if m > 0:
                    lh[:m, :, j].copy_(conds[u][:, :, first:first + m].permute(2, 1, 0))
            eng.set_conditioning(lh, 0, n)
            eng.set_selectors_random_stream(seeds[b0], first, n)
            eng.run_stream(first, n, SLOTS)
            eng.get_yout(stage, 0, n)
            for j, u in enumerate(batch):
                m = min(n, conds[u].size(2) - first)
                if m > 0:
                    outs[u][first:first + m].copy_(stage[j, :m])
    torch.cuda.synchronize()
    return outs


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", default=None, help="directory for serve_bench.json")
    ap.add_argument("--utterances", type=int, default=256)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    for k in ("NVWN_FP16_KERNEL", "NVWN_LAT_CLUSTER", "NVWN_LAT_MAX_B", "NVWN_TC_TILE", "NVWN_TC_NODUP", "NVWN_TC_FUSED"):
        os.environ.pop(k, None)

    rng = np.random.default_rng(args.seed)
    frames = [int(v) for v in rng.integers(LO // STRIDE, HI // STRIDE + 1, args.utterances)]
    lengths = [STRIDE * t for t in frames]
    offsets = [int(v) for v in rng.integers(0, HI + 1, args.utterances)]
    seeds = [int(v) for v in rng.integers(0, 2 ** 62, args.utterances)]
    g = torch.Generator(device="cuda").manual_seed(args.seed)
    base = 0.5 * torch.randn((2 * R, L, 2 * HI + 1), generator=g, device="cuda")
    conds = [base[:, :, o:o + n] for o, n in zip(offsets, lengths)]
    mels = [torch.randn((MEL, t), generator=g, device="cuda") for t in frames]
    cnet = conditioning_network(args.seed)
    net = network(args.seed)
    info = card()

    useful = sum(lengths)
    padded = sum(SLOTS * max(lengths[b:b + SLOTS]) for b in range(0, len(lengths), SLOTS))
    plan = plan_slots(lengths, SLOTS, WINDOW)
    steps = max(t + n for (_, t), n in zip(plan, lengths))

    # warm-up: engine creation, weight upload and first launches of both arms
    net.infer_many([c[:, :, :2 * WINDOW] for c in conds[:SLOTS]], seeds[:SLOTS], slots=SLOTS, window=WINDOW, fp16=True)
    static_batches(net, [c[:, :, :WINDOW] for c in conds[:SLOTS]], seeds[:SLOTS])
    net.infer_many_from_features([m[:, :2 * WINDOW // STRIDE] for m in mels[:SLOTS]], seeds[:SLOTS], *cnet, STRIDE, slots=SLOTS,
                                 window=WINDOW, fp16=True)

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    timing = {}
    cont = net.infer_many(conds, seeds, slots=SLOTS, window=WINDOW, fp16=True, timing=timing)
    t_cont = time.perf_counter() - t0
    launch = net._engine(SLOTS, WINDOW, True).launch_info()

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mtiming = {}
    mel = net.infer_many_from_features(mels, seeds, *cnet, STRIDE, slots=SLOTS, window=WINDOW, fp16=True, timing=mtiming)
    t_mel = time.perf_counter() - t0
    windows = (steps + WINDOW - 1) // WINDOW

    t0 = time.perf_counter()
    stat = static_batches(net, conds, seeds)
    t_stat = time.perf_counter() - t0
    del cont, stat, mel
    split = production_split(net, mels, cnet)
    after = card()
    cond_bytes = sum(lengths) * 2 * R * L * 4

    res = {
        "workload": {"model": "C3", "dtype": "fp16", "slots": SLOTS, "window": WINDOW, "utterances": args.utterances,
                     "lengths": [LO, HI], "seed": args.seed, "useful_samples": useful},
        "card": info, "card_after": after, "launch": {k: launch[k] for k in ("kernel", "grid", "batch_per_cta", "cluster")},
        "continuous": {"seconds": t_cont, "useful_samples_per_s": useful / t_cont, "steps": steps,
                       "idle_slot_fraction": 1.0 - useful / (SLOTS * steps),
                       "restart_upload_s": timing.get("restart_upload_s"), "generate_s": timing.get("generate_s")},
        "mel": {"seconds": t_mel, "useful_samples_per_s": useful / t_mel, "windows": windows, **mtiming,
                "produce_ms_per_window": 1e3 * mtiming["produce_s"] / windows,
                "produce_wait_ms_per_window": 1e3 * mtiming["produce_wait_s"] / windows,
                "produce_hidden_fraction": 1.0 - mtiming["produce_wait_s"] / mtiming["produce_s"]},
        "static": {"seconds": t_stat, "useful_samples_per_s": useful / t_stat, "padding_fraction": 1.0 - useful / padded},
        "speedup": t_stat / t_cont,
        "mel_vs_continuous": t_cont / t_mel,
        "input_bytes": {"continuous": cond_bytes, "static": cond_bytes, "mel": sum(frames) * MEL * 4},
        "production_alone": split,
    }
    line = json.dumps(res)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "serve_bench.json"), "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
