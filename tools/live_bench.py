"""Live vocoding (NVWaveNet.open_live): mel frames pushed one at a time, each push generating the samples its frame completes.

C3 model (fp16, L20, R64/S256/A256, maxDilation 512), C = 80 mel channels, upsampling window 800, stride 200, so one frame is
12.5 ms of 16 kHz audio.  Per batch size (1 and 64 by default) and per pacing:
  * fast: every frame is there from the start, pushed as soon as the last push returned;
  * paced: frame i arrives at 12.5 ms * i after the first, as from an acoustic model running at real time, and is pushed then.
Per push the time from the call to its samples being on the host (push, then a copy to host memory); the first push's time is
the first-audio latency.  The real-time factor is the audio's duration over the time from the first push to the last samples on
the host.  The total time is set against infer_many_from_features of the same finished frames on as many slots (its engine created
and warmed up first), and for batch 1, where both draw the same selectors, the samples are compared bit for bit.  The card's name
and power limit are read in the same process.  Prints one JSON object; --out also writes it to a file.

    python tools/live_bench.py [--frames 160] [--batches 1,64] [--window 4096] [--out result.json]
"""
import argparse
import json
import os
import subprocess
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

L, R, S, A, MAXDIL = 20, 64, 256, 256, 512
C, KW, STRIDE, RATE = 80, 800, 200, 16000
FRAME_S = STRIDE / RATE
SEED = 4321


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    res = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [v.strip() for v in res.stdout.splitlines()[0].split(",")])) if res.returncode == 0 else {}


def stats(v):
    v = np.asarray(v) * 1e3
    return {"mean_ms": float(v.mean()), "p50_ms": float(np.percentile(v, 50)), "p90_ms": float(np.percentile(v, 90)),
            "p99_ms": float(np.percentile(v, 99)), "max_ms": float(v.max())}


def live_run(wnet, cnet, frames, window, paced):
    """one session over frames [B][C][T], one frame per push; returns the result dict and the samples [B][T * stride] (host)"""
    B, _, T = frames.shape
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    live = wnet.open_live(*cnet, STRIDE, B, SEED, window=window, fp16=True)
    torch.cuda.synchronize()
    open_s = time.perf_counter() - t0
    lat, lag, ys = [], [], []
    start = time.perf_counter()
    for i in range(T):
        arrival = start + i * FRAME_S
        if paced:
            while time.perf_counter() < arrival:
                time.sleep(max(0.0, min(arrival - time.perf_counter(), 1e-3)))
        t = time.perf_counter()
        y = live.push(frames[:, :, i:i + 1]).cpu()
        done = time.perf_counter()
        lat.append(done - t)
        lag.append(done - arrival)
        ys.append(y.numpy())
    total = time.perf_counter() - start
    live.close()
    audio_s = T * FRAME_S
    out = {"open_s": open_s, "first_audio_ms": lat[0] * 1e3, "push_to_host": stats(lat), "total_s": total, "audio_s": audio_s,
           "real_time_factor": audio_s / total}
    if paced:
        out["behind_arrival"] = stats(lag)                             # last samples on the host after their frame arrived
    return out, np.concatenate(ys, axis=1)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--frames", type=int, default=160, help="frames per utterance (2 s of audio)")
    ap.add_argument("--batches", default="1,64")
    ap.add_argument("--window", type=int, default=4096)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available() or nw._lib.lib().nvwn_device_count() == 0:
        sys.exit("live_bench: no CUDA device")
    w = refgen.lively_inputs(SEED, R, S, A, L, 1, 1)
    wnet = _net(w, L, R, S, A, MAXDIL)
    g = torch.Generator(device="cuda"); g.manual_seed(SEED)
    rnd = lambda *shape, s=1.0: torch.randn(shape, generator=g, device="cuda", dtype=torch.float32) * s
    cnet = (rnd(C, C, KW, s=0.02), rnd(C, s=0.01), rnd(L * 2 * R, C, s=0.05), rnd(L * 2 * R, s=0.05))
    result = {"model": "C3", "channels": C, "upsample_window": KW, "stride": STRIDE, "rate_hz": RATE, "frames": args.frames,
              "window": args.window, "card": card(), "runs": []}
    for B in [int(v) for v in args.batches.split(",")]:
        frames = rnd(B, C, args.frames).cpu().numpy()               # host frames, as an acoustic model hands them over
        live_run(wnet, cnet, frames[:, :, :8], args.window, False)   # warm-up: modules, allocator, engine creation
        fast, y_live = live_run(wnet, cnet, frames, args.window, False)
        paced, _ = live_run(wnet, cnet, frames, args.window, True)
        feats = [torch.from_numpy(np.ascontiguousarray(frames[b])) for b in range(B)]
        seeds = [SEED] * B
        many = lambda: wnet.infer_many_from_features(feats, seeds, *cnet, STRIDE, slots=B, window=args.window, fp16=True)
        many()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        outs = many()
        y_many = np.stack([o.cpu().numpy() for o in outs])
        many_s = time.perf_counter() - t0
        run = {"batch": B, "fast": fast, "paced": paced, "infer_many_from_features_s": many_s,
               "live_fast_over_many": fast["total_s"] / many_s}
        if B == 1:
            run["bit_equal_to_infer_many"] = bool(np.array_equal(y_live, y_many))
        result["runs"].append(run)
        print(json.dumps(run), flush=True)
    text = json.dumps(result)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
