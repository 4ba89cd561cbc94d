"""Multi-model serving (nvwn_set_model, ModelSet): several models of one shape in one engine.

C3 model shape (fp16, L20, R64/S256/A256, maxDilation 512), seeded weights per model, 64 slots, so G = 8 rows per model group on the
8-row cluster kernel and up to 8 models per engine.
  * fixed batch: samples/s of a 64-slot engine generating --fixed-samples samples in windows of 4 096 with no group table, and
    of one holding eight models with V = 1, 2, 4 and 8 of them spread over its groups (group g runs model g mod V); the arms
    alternated over --rounds rounds, reported as medians with the spread;
  * queue: --utterances utterances, lengths uniform in [16 000, 160 000], model drawn uniformly from V = 4, seeded.  Three arms,
    alternated over --rounds rounds, reported as medians with the spread: ModelSet.infer_many on one 64-slot engine; one 64-slot
    engine per model (NVWaveNet.infer_many), each running its own queue one after another; and the same per-model engines run
    concurrently, one CUDA stream and host thread each.  Every arm's outputs are compared with the sequential arm's bit for bit.
The device bytes of each arm's engines are computed from their shapes.  The card's name, power limit and SM clock are read in
the same process.  Prints one JSON object with everything; --out DIR also writes it to DIR/model_bench.json.

    python tools/model_bench.py [--utterances 256] [--rounds 3] [--out DIR]
"""
import argparse
import json
import os
import statistics
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import nv_wavenet_b200 as nw  # noqa: E402
from nv_wavenet_b200.nv_wavenet import ModelSet  # noqa: E402
from tests import refgen  # noqa: E402
from tests.test_gpu_zz_selectors import _net  # noqa: E402
from tools.live_bench import card  # noqa: E402

L, MAXDIL, R, S, A = 20, 512, 64, 256, 256
SLOTS, WINDOW = 64, 4096


def engine_bytes(models, slots=SLOTS, window=WINDOW):
    """Device bytes of one fp16 latency-family engine of `slots` rows and `window` samples holding `models` models, from shapes: the
    conditioning store and selectors, yOut and forced indices, the history ring, the fp32 staging buffer, and per model the weight
    blob and the packed image (taken as the blob's size again)."""
    tiles = (slots + 15) // 16 * 16
    store = window * L * tiles * 2 * R * 2
    ring = (MAXDIL + 1) * L * tiles * R * 2
    per_row = window * (4 + 4 + 4)                                  # selectors, yOut, forced
    blob = 2 * (2 * A * R + L * (2 * 2 * R * R + R * R + S * R + 2 * R + R + S) + A * S + A * A + 2 * A)
    stage = max(L * slots * 2 * R, 16 << 20) * 4
    return store + ring + slots * per_row + stage + models * 2 * blob


def fixed_batch(wnets, rounds, samples):
    """samples/s of a 64-slot engine with no group table, and of one holding all the nets as models with V = 1, 2, 4 and 8 of them
    spread over its groups (group g runs model g mod V); the arms alternated over `rounds` rounds.  Returns (G, {arm: rates})."""
    plain, multi = ModelSet(wnets[:1]), ModelSet(wnets)
    engines = {"no_table": plain._engine(SLOTS, WINDOW, True), "table": multi._engine(SLOTS, WINDOW, True)}
    G = engines["table"].model_group
    n_groups = (SLOTS + G - 1) // G
    arms = {"V1_no_table": ("no_table", None)}
    arms.update({f"V{V}": ("table", [g % V for g in range(n_groups)]) for V in (1, 2, 4, 8) if V <= min(n_groups, len(wnets))})
    g = torch.Generator(device="cuda").manual_seed(5)
    lh = 0.5 * torch.randn((WINDOW, L, SLOTS, 2 * R), generator=g, device="cuda")
    for eng in engines.values():
        eng.set_conditioning(lh, 0, WINDOW)

    def run(arm, n):
        key, table = arms[arm]
        eng = engines[key]
        eng.reset_history()
        if table is not None:
            eng.set_group_models(table)
        for first in range(0, n, WINDOW):
            m = min(WINDOW, n - first)
            eng.set_selectors_random_stream(7, first, m)
            eng.run_stream(first, m, SLOTS)

    for arm in arms:                                                # warm-up: modules, packs
        run(arm, WINDOW)
    rates, info = {arm: [] for arm in arms}, {}
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(rounds):
        for arm in arms:
            torch.cuda.synchronize()
            a.record()
            run(arm, samples)
            b.record()
            torch.cuda.synchronize()
            rates[arm].append(SLOTS * samples / (a.elapsed_time(b) / 1e3))
            info[arm] = engines[arms[arm][0]].launch_info()
    plain.close()
    multi.close()
    return G, rates, info


def spread(v):
    return {"median": statistics.median(v), "min": min(v), "max": max(v), "runs": v}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utterances", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--fixed-samples", type=int, default=8 * WINDOW)
    ap.add_argument("--min-len", type=int, default=16000)
    ap.add_argument("--max-len", type=int, default=160000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("model_bench needs a CUDA device")
    out = {"card": card(), "shape": dict(L=L, R=R, S=S, A=A, max_dilation=MAXDIL, slots=SLOTS, window=WINDOW, dtype="fp16")}
    wnets = [_net(refgen.lively_inputs(1000 + m, R, S, A, L, 1, 1), L, R, S, A, MAXDIL) for m in range(8)]

    # ---- fixed batch
    G, rates, info = fixed_batch(wnets, args.rounds, args.fixed_samples)
    base = statistics.median(rates["V1_no_table"])
    fixed = {"group_rows": G, "rounds": args.rounds}
    for arm, v in rates.items():
        fixed[arm] = {"samples_per_s": spread(v), "median_vs_no_table": statistics.median(v) / base, "launch": info[arm]}
    out["fixed_batch"] = fixed
    print(json.dumps({"fixed_batch": fixed}), flush=True)

    # ---- queue
    V = 4
    rng = np.random.default_rng(2024)
    n = args.utterances
    lengths = [int(v) for v in rng.integers(args.min_len, args.max_len + 1, n)]
    models = [int(v) for v in rng.integers(0, V, n)]
    seeds = [int(v) for v in rng.integers(0, 2 ** 62, n)]
    offsets = [int(v) for v in rng.integers(0, 20000, n)]
    g = torch.Generator(device="cuda").manual_seed(2025)
    base = 0.5 * torch.randn((2 * R, L, args.max_len + 20000), generator=g, device="cuda", dtype=torch.float32)
    conds = [base[:, :, o:o + m] for o, m in zip(offsets, lengths)]
    ms = ModelSet(wnets[:V])
    ms._engine(SLOTS, WINDOW, True)                                 # every arm's engines exist before the first timed run
    for m in range(V):
        wnets[m]._engine(SLOTS, WINDOW, True)
    mine = [[u for u in range(n) if models[u] == m] for m in range(V)]

    def one_engine():
        return ms.infer_many(models, conds, seeds, slots=SLOTS, window=WINDOW, fp16=True)

    def serve_model(m, outs):
        got = wnets[m].infer_many([conds[u] for u in mine[m]], [seeds[u] for u in mine[m]], slots=SLOTS, window=WINDOW, fp16=True)
        for u, o in zip(mine[m], got):
            outs[u] = o

    def per_model():
        outs = [None] * n
        for m in range(V):
            serve_model(m, outs)
        return outs

    streams = [torch.cuda.Stream() for _ in range(V)]

    def per_model_concurrent():
        outs, errors = [None] * n, []

        def worker(m):
            try:
                with torch.cuda.stream(streams[m]):
                    serve_model(m, outs)
                streams[m].synchronize()
            except BaseException as exc:                            # re-raised on the main thread
                errors.append(exc)

        threads = [threading.Thread(target=worker, args=(m,)) for m in range(V)]
        for th in threads:
            th.start()
        for th in threads:
            th.join()
        if errors:
            raise errors[0]
        return outs

    arms = {"modelset_one_engine": one_engine, "engine_per_model_sequential": per_model,
            "engine_per_model_concurrent": per_model_concurrent}
    times = {k: [] for k in arms}
    results = {}
    for r in range(args.rounds):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = fn()
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
            if r == 0:
                results[k] = [o.cpu() for o in res]
            del res
    ref = results["engine_per_model_sequential"]
    same = {k: all(torch.equal(a, b) for a, b in zip(v, ref)) for k, v in results.items()}
    total = sum(lengths)
    queue = {"utterances": n, "models": V, "samples": total, "rounds": args.rounds, "outputs_bit_identical_to_sequential": same}
    for k, ts in times.items():
        med = statistics.median(ts)
        queue[k] = {"median_s": med, "min_s": min(ts), "max_s": max(ts), "samples_per_s": total / med, "runs_s": ts}
    queue["modelset_one_engine"]["device_bytes"] = engine_bytes(V)
    queue["engine_per_model_sequential"]["device_bytes"] = V * engine_bytes(1)
    queue["engine_per_model_concurrent"]["device_bytes"] = V * engine_bytes(1)
    for k in ("engine_per_model_sequential", "engine_per_model_concurrent"):
        queue[f"one_engine_speedup_vs_{k}"] = queue[k]["median_s"] / queue["modelset_one_engine"]["median_s"]
    out["queue"] = queue
    out["card_after"] = card()
    print(json.dumps(out), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "model_bench.json"), "w") as f:
            json.dump(out, f, indent=1)
    ms.close()
    for net in wnets:
        for eng in net._engines.values():
            eng.close()
        net._engines.clear()


if __name__ == "__main__":
    main()
