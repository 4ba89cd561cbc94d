"""Prompted live streams (LivePool.open(seed, prompt=)): how long a stream that continues given audio waits for its first sample.

C3 model (fp16, L20, R64/S256/A256, maxDilation 512), C = 80 mel channels, upsampling window 800, stride 200 (16 kHz), a pool of 64
slots and a window of 800 samples.  Per prompt length (0.5, 1 and 2 s by default) and per number of streams opened together (1 and
64): every stream's frames (its prompt's and 0.4 s more) are pushed right after open(), then step() runs until every stream has
all its samples.  Reported: the time from the first open() to each stream's first generated samples on the host (p50 and max); the
GPU time of the prompt stage (the scoring engine's producer load and runs, the scoring and the state saves, CUDA events around each
scoring stream) and of the loads into the pool's slots.  Baseline: the same prompt forced through generation on a batch-1 engine
(nvwn_set_forced, conditioning from the same frames), the only other way to a generation state at sample P; its GPU time per
prompt (CUDA events).  The card's name and power limit are read in the same process.  One run per arm.  Prints one JSON object per
arm and one with everything; --out DIR also writes the last to DIR/live_prompt_bench.json.

    python tools/live_prompt_bench.py [--seconds 0.5,1,2] [--streams 1,64] [--out DIR]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import nv_wavenet_b200 as nw  # noqa: E402
from tests import refgen  # noqa: E402
from tests.test_gpu_zz_selectors import _net  # noqa: E402
from tools.live_bench import C, KW, L, MAXDIL, RATE, A, R, S, STRIDE, SEED, card  # noqa: E402

SLOTS, WINDOW, TAIL_FRAMES = 64, 800, 32


def pool_run(wnet, cnet, frames, prompts):
    """opens len(frames) prompted streams, pushes all their frames and steps until they are done"""
    pool = wnet.open_live_pool(*cnet, STRIDE, SLOTS, WINDOW, fp16=True, timed=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ids = [pool.open(SEED + s, prompts[s]) for s in range(len(frames))]
    for i, f in zip(ids, frames):
        pool.push(i, f)
        pool.finish(i)
    first, out = {}, {i: [] for i in ids}
    while pool._streams:
        for i, y in pool.step().items():
            out[i].append(y.cpu().numpy())
            first.setdefault(i, time.perf_counter() - t0)
    prompt_s = pool.prompt_seconds()
    _, load_s = pool.state_seconds()
    pool.close()
    v = np.array([first[i] for i in ids]) * 1e3
    return [np.concatenate(out[i]) for i in ids], {"open_to_first_sample_p50_ms": float(np.percentile(v, 50)), "open_to_first_sample_max_ms":
                                                   float(v.max()), "prompt_stage_gpu_ms": prompt_s * 1e3, "load_gpu_ms": load_s * 1e3}


def forced_run(cnet, w, frames, prompt):
    """the prompt forced through generation on a batch-1 engine: GPU ms of conditioning and generation of its P samples"""
    P = prompt.shape[0]
    eng = nw.NVWavenetInfer(L, MAXDIL, 1, P, R=R, S=S, A=A, dtype=nw.FP16)
    eng.load(w)
    eng.set_forced(np.ascontiguousarray(prompt[None], np.int32))
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for rep in range(2):                                            # the first is a warm-up
        eng.reset_history()
        ev[0].record()
        eng.cond_producer_load(frames[None, :, :(P - 1) // STRIDE + 1], *cnet, STRIDE)
        eng.cond_producer_run(0, P)
        eng.set_selectors_random(SEED)
        eng.run(P, 1)
        ev[1].record()
    torch.cuda.synchronize()
    eng.close()
    return ev[0].elapsed_time(ev[1])


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--seconds", default="0.5,1,2", help="prompt lengths in seconds")
    ap.add_argument("--streams", default="1,64")
    ap.add_argument("--out", default=None, help="directory for live_prompt_bench.json")
    args = ap.parse_args()
    if not torch.cuda.is_available() or nw._lib.lib().nvwn_device_count() == 0:
        sys.exit("live_prompt_bench: no CUDA device")
    w = refgen.lively_inputs(SEED, R, S, A, L, 1, 1)
    wnet = _net(w, L, R, S, A, MAXDIL)
    g = torch.Generator(device="cuda"); g.manual_seed(SEED)
    rnd = lambda *shape, s=1.0: torch.randn(shape, generator=g, device="cuda", dtype=torch.float32) * s
    cnet = tuple(t.cpu().numpy() for t in (rnd(C, C, KW, s=0.02), rnd(C, s=0.01), rnd(L * 2 * R, C, s=0.05), rnd(L * 2 * R, s=0.05)))
    lengths = [int(round(float(v) * RATE)) for v in args.seconds.split(",")]
    counts = [int(v) for v in args.streams.split(",")]
    n_max = max(counts)
    frames_all = rnd(n_max, C, max(lengths) // STRIDE + TAIL_FRAMES).cpu().numpy()
    codes_all = np.random.default_rng(SEED).integers(0, A, (n_max, max(lengths))).astype(np.int32)
    result = {"model": "C3", "channels": C, "upsample_window": KW, "stride": STRIDE, "rate_hz": RATE, "slots": SLOTS, "window": WINDOW,
              "tail_frames": TAIL_FRAMES, "card": card(), "arms": []}
    pool_run(wnet, cnet, [frames_all[0, :, :8]], [codes_all[0, :400]])          # warm-up: modules, allocator, the scoring engine
    for P in lengths:
        T = (P - 1) // STRIDE + 1 + TAIL_FRAMES
        forced_ms = forced_run(cnet, w, frames_all[0], codes_all[0, :P])
        for n in counts:
            frames = [np.ascontiguousarray(frames_all[s, :, :T]) for s in range(n)]
            ys, res = pool_run(wnet, cnet, frames, [codes_all[s, :P] for s in range(n)])
            arm = {"prompt_samples": P, "prompt_s": P / RATE, "streams": n, **res, "forced_batch1_gpu_ms_per_prompt": forced_ms,
                   "generated_samples_per_stream": int(ys[0].size)}
            result["arms"].append(arm)
            print(json.dumps(arm), flush=True)
    text = json.dumps(result)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "live_prompt_bench.json"), "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
