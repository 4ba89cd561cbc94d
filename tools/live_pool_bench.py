"""Live serving (NVWaveNet.open_live_pool): many live streams, each with its own frames arriving at its own pace, in one engine's slots.

C3 model (fp16, L20, R64/S256/A256, maxDilation 512), C = 80 mel channels, upsampling window 800, stride 200, so one frame is
12.5 ms of 16 kHz audio.  A pool of 64 slots, per launch window (200 and 800 samples by default), per stream count (64 and 128)
and per pacing:
  * paced: stream s's frame i arrives at 12.5 ms * i after the stream's start (starts spread over the first 50 ms), with seeded
    jitter of up to 2 ms, and one stream in eight stalls once for 100 ms at a random frame;
  * fast: every frame is there from the start.
One thread pushes every arrived frame and calls step() until every stream is done.  Per arm: the first-audio latency (a stream's
first frame arriving to its first samples on the host), the frame-to-host lag (the last frame a piece of samples reads arriving to
that piece on the host) at p50, p99 and max, the real-time factor (all streams' audio over the wall time), the launches, parks and
resumes, and the GPU time of the saves and loads (CUDA events).  The baseline is the same streams, each in its own
open_live(batch_size=1) session with the same window, pushed round-robin from the same thread; every stream's samples are compared
with the baseline's bit for bit.  The card's name and power limit are read in the same process.  Prints one JSON object per arm
and one with everything; --out DIR also writes the last to DIR/live_pool_bench.json.

    python tools/live_pool_bench.py [--frames 64] [--windows 200,800] [--streams 64,128] [--out DIR]
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
from tools.live_bench import C, FRAME_S, KW, L, MAXDIL, RATE, A, R, S, STRIDE, SEED, card  # noqa: E402

SLOTS = 64


def arrivals(n_streams, frames, paced, seed):
    """[stream][frame] arrival times in seconds from the start"""
    if not paced:
        return np.zeros((n_streams, frames))
    rng = np.random.default_rng(seed)
    start = rng.uniform(0, 0.05, n_streams)[:, None]
    t = start + np.arange(frames)[None, :] * FRAME_S + rng.uniform(0, 0.002, (n_streams, frames))
    for s in range(0, n_streams, 8):                                 # one stream in eight stalls once for 100 ms
        t[s, int(rng.integers(1, frames)):] += 0.1
    return np.maximum.accumulate(t, axis=1)


def pct(v):
    v = np.asarray(v) * 1e3
    return {"p50_ms": float(np.percentile(v, 50)), "p99_ms": float(np.percentile(v, 99)), "max_ms": float(v.max())}


def drive(frames, arrive, open_stream, push, finish, poll):
    """the one-thread loop both servers share: pushes every arrived frame, then poll() -> [(stream, samples [k] on the host)]"""
    n, T = arrive.shape
    given = [0] * n
    out = [[] for _ in range(n)]
    first, lag, done_at = [None] * n, [], 0.0
    handles = [open_stream(s) for s in range(n)]
    produced = [0] * n
    start = time.perf_counter()
    while True:
        now = time.perf_counter() - start
        for s in range(n):
            k = int(np.searchsorted(arrive[s], now, side="right")) - given[s]
            if k > 0:
                push(handles[s], frames[s][:, given[s]:given[s] + k])
                given[s] += k
                if given[s] == T:
                    finish(handles[s])
        got = poll(handles)
        t = time.perf_counter() - start
        for s, y in got:
            if first[s] is None:
                first[s] = t - arrive[s][0]
            produced[s] += len(y)
            lag.append(t - arrive[s][(produced[s] - 1) // STRIDE])
            out[s].append(y)
            done_at = t
        if all(p == T * STRIDE for p in produced):
            break
        if not got and min(given) < T:
            nxt = min(arrive[s][given[s]] for s in range(n) if given[s] < T)
            time.sleep(max(0.0, min(nxt - (time.perf_counter() - start), 1e-3)))
    audio = n * T * FRAME_S
    return [np.concatenate(o) for o in out], {"first_audio": pct(first), "frame_to_host_lag": pct(lag), "wall_s": done_at,
                                               "real_time_factor": audio / done_at}


def pool_run(wnet, cnet, frames, arrive, window):
    pool = wnet.open_live_pool(*cnet, STRIDE, SLOTS, window, fp16=True, timed=True)
    ys, res = drive(frames, arrive, lambda s: pool.open(SEED + s), pool.push, pool.finish,
                    lambda h: [(h.index(i), y.cpu().numpy()) for i, y in pool.step().items()])
    save_s, load_s = pool.state_seconds()
    res.update(launches=pool.launches, parks=pool.parks, resumes=pool.resumes, save_gpu_ms=save_s * 1e3, load_gpu_ms=load_s * 1e3)
    pool.close()
    return ys, res


def session_run(wnet, cnet, frames, arrive, window):
    sessions = [wnet.open_live(*cnet, STRIDE, 1, SEED + s, window=window, fp16=True) for s in range(len(frames))]
    pending = {}

    def push(h, f):
        y = sessions[h].push(f[None])
        if y.shape[1]:
            pending.setdefault(h, []).append(y)

    def poll(h):
        out = [(s, torch.cat(ys, dim=1)[0].cpu().numpy()) for s, ys in pending.items()]
        pending.clear()
        return out

    ys, res = drive(frames, arrive, lambda s: s, push, lambda h: None, poll)
    for x in sessions:
        x.close()
    return ys, res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--frames", type=int, default=64, help="frames per stream (0.8 s of audio)")
    ap.add_argument("--windows", default="200,800")
    ap.add_argument("--streams", default="64,128")
    ap.add_argument("--out", default=None, help="directory for live_pool_bench.json")
    args = ap.parse_args()
    if not torch.cuda.is_available() or nw._lib.lib().nvwn_device_count() == 0:
        sys.exit("live_pool_bench: no CUDA device")
    w = refgen.lively_inputs(SEED, R, S, A, L, 1, 1)
    wnet = _net(w, L, R, S, A, MAXDIL)
    g = torch.Generator(device="cuda"); g.manual_seed(SEED)
    rnd = lambda *shape, s=1.0: torch.randn(shape, generator=g, device="cuda", dtype=torch.float32) * s
    cnet = tuple(t.cpu().numpy() for t in (rnd(C, C, KW, s=0.02), rnd(C, s=0.01), rnd(L * 2 * R, C, s=0.05), rnd(L * 2 * R, s=0.05)))
    result = {"model": "C3", "channels": C, "upsample_window": KW, "stride": STRIDE, "rate_hz": RATE, "frames": args.frames, "slots": SLOTS,
              "card": card(), "arms": []}
    n_max = max(int(v) for v in args.streams.split(","))
    frames_all = rnd(n_max, C, args.frames).cpu().numpy()
    warm = frames_all[:4, :, :8]
    pool_run(wnet, cnet, warm, arrivals(4, 8, False, 0), 200)          # warm-up: modules, allocator
    session_run(wnet, cnet, warm, arrivals(4, 8, False, 0), 200)
    for window in [int(v) for v in args.windows.split(",")]:
        for n in [int(v) for v in args.streams.split(",")]:
            for paced in (True, False):
                frames = list(frames_all[:n])
                arrive = arrivals(n, args.frames, paced, 17 + n)
                y_pool, pool = pool_run(wnet, cnet, frames, arrive, window)
                y_one, one = session_run(wnet, cnet, frames, arrive, window)
                arm = {"window": window, "streams": n, "pacing": "paced" if paced else "fast", "pool": pool, "sessions": one,
                       "bit_equal": all(np.array_equal(a, b) for a, b in zip(y_pool, y_one))}
                result["arms"].append(arm)
                print(json.dumps(arm), flush=True)
    text = json.dumps(result)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "live_pool_bench.json"), "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
