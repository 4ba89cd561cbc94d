"""Long-form generation through a fixed-size engine (nvwn_run_stream), against one engine that holds the whole length.

C3 model (fp16, L20, R64/S256/A256, maxDilation 512), B = 64 utterances of 160 000 samples by default.  Conditioning comes from
the device producer (mel frames, ConvTranspose1d(80, 80, 800, 200) + 1x1 projection):
  * single: one engine of N = 160 000 (its conditioning store alone is ~52 GB), filled in one call, generated in one nvwn_run;
  * chunked: the same engine and data generated in nvwn_run_partial chunks of 2 000 samples, so the per-launch cost of restarting
    the kernel's pipelines is (chunked - single) / (chunk launches - 1);
  * window W: an engine of N = W; the producer fills half a window on a side stream while the other half is generated
    (run_stream per half window, each waiting on an event), yOut read back per chunk.
Per run: samples/s (utterance samples, B x length / time), device bytes of the engine (free memory before and after creating it),
engine launches, and whether yOut is bit-equal to the single engine's.  The card's name, power limit and clocks are read in the same
process.  Prints one JSON object; --out also writes it to a file.

    python tools/stream_bench.py [--samples 160000] [--windows 2000,4000,16000] [--out result.json]
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
from nv_wavenet_b200 import _lib  # noqa: E402
from tests import refgen  # noqa: E402

L, R, S, A, MAXDIL = 20, 64, 256, 256, 512
C, KW, STRIDE = 80, 800, 200
SEED = 1234


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    res = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [v.strip() for v in res.stdout.splitlines()[0].split(",")])) if res.returncode == 0 else {}


def free_bytes():
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


def make_engine(n, B, w):
    before = free_bytes()
    e = nw.NVWavenetInfer(L, MAXDIL, B, n, R=R, S=S, A=A, dtype=nw.FP16)
    used = before - free_bytes()
    e.load(w)
    return e, used


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--samples", type=int, default=160000)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--windows", default="2000,4000,16000")
    ap.add_argument("--chunk", type=int, default=2000, help="run_partial chunk of the per-launch measurement")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available() or nw._lib.lib().nvwn_device_count() == 0:
        sys.exit("stream_bench: no CUDA device")
    B = args.batch
    frames = args.samples // STRIDE
    N = frames * STRIDE
    w = refgen.lively_inputs(SEED, R, S, A, L, 1, 1)
    g = torch.Generator(device="cuda"); g.manual_seed(SEED)
    rnd = lambda *shape, s=1.0: torch.randn(shape, generator=g, device="cuda", dtype=torch.float32) * s
    cond = (rnd(B, C, frames), rnd(C, C, KW, s=0.02), rnd(C, s=0.01), rnd(L * 2 * R, C, s=0.05), rnd(L * 2 * R, s=0.05), STRIDE)
    result = {"model": "C3", "batch": B, "samples": N, "card": card()}

    # ---- one engine of the whole length
    e, used = make_engine(N, B, w)
    e.reset_history(); e.set_conditioning_from_features(*cond); e.set_selectors_random(SEED)
    _lib.check(e._l.nvwn_run_partial(e._h, 0, 200, N, B, None, 0, None), "warm-up")
    l0 = e.launch_info()["launches"]
    e.reset_history()
    t = timed(lambda: e.run(N, B))
    y_single = np.zeros((B, N), np.int32); e.get_yout(y_single, 0, N); e.synchronize()
    result["single"] = {"engine_bytes": used, "seconds": t, "samples_per_s": B * N / t, "khz_per_utterance": N / t / 1e3,
                        "launches": e.launch_info()["launches"] - l0}

    def chunked():
        for init in range(0, N, args.chunk):
            _lib.check(e._l.nvwn_run_partial(e._h, init, min(args.chunk, N - init), N, B, None, 0, None), "run_partial")
    e.reset_history()
    l0 = e.launch_info()["launches"]
    tc = timed(chunked)
    launches = e.launch_info()["launches"] - l0
    y = np.zeros((B, N), np.int32); e.get_yout(y, 0, N); e.synchronize()
    result["chunked"] = {"chunk": args.chunk, "seconds": tc, "samples_per_s": B * N / tc, "launches": launches,
                         "bit_equal": bool(np.array_equal(y, y_single)),
                         "per_launch_restart_us": (tc - t) / (launches - 1) * 1e6 if launches > 1 else None}
    e.close()
    del e

    # ---- windows
    result["windows"] = []
    for W in [int(v) for v in args.windows.split(",")]:
        e, used = make_engine(W, B, w)
        assert e.cond_producer_load(*cond) == N
        side, gen = torch.cuda.Stream(), torch.cuda.Stream()
        out = torch.empty((B, N), dtype=torch.int32, device="cuda")
        half = max(1, W // 2)

        def go(total):
            e.reset_history()
            done = []
            for k, first in enumerate(range(0, total, half)):
                n = min(half, total - first)
                if k >= 2:
                    side.wait_event(done[k - 2])           # the chunk whose positions this one overwrites is generated and read
                e.cond_producer_run_stream(first, n, stream=side)
                ready = torch.cuda.Event(); ready.record(side)
                gen.wait_event(ready)
                e.set_selectors_random_stream(SEED, first, n, stream=gen)
                e.run_stream(first, n, B, stream=gen)
                e.get_yout_stream(out[:, first:first + n], first, n, stream=gen)
                done.append(torch.cuda.Event()); done[-1].record(gen)
        go(min(N, 2 * half))                                # warm-up
        l0 = e.launch_info()["launches"]
        tw = timed(lambda: go(N))
        result["windows"].append({"window": W, "engine_bytes": used, "seconds": tw, "samples_per_s": B * N / tw,
                                  "khz_per_utterance": N / tw / 1e3, "launches": e.launch_info()["launches"] - l0,
                                  "bit_equal": bool(np.array_equal(out.cpu().numpy(), y_single))})
        e.close()
        del e
    result["card_after"] = card()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
