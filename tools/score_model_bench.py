"""Scoring by model (nvwn_set_score_models, ModelSet.infer_many(prompts=)): what it costs to score rows with several models in one
engine.

Two model shapes, fp16, seeded weights per model: C3 (L20, R64/S256/A256, maxDilation 512) and R128 L30 (S256/A256, maxDilation 512).
For each, seeded audio and conditioning of 64 rows x 4 096 samples:
  (a) one engine holding eight models scores the rows with an all-zero table (the one-model scorer), and with V = 2, 4 and 8 models
      over the rows (row b runs model b mod V);
  (b) V one-model engines of 64 / V rows each score their own rows, one after another;
and for the C3 shape
  (c) a prompted queue of --utterances utterances over four models: ModelSet.infer_many(prompts=) on one 64-slot engine against each
      net's NVWaveNet.infer_many(prompts=) of its own utterances, run one after another.
Each arm gets a warm-up call and then five timed calls, the arms alternating call by call; times are CUDA events around each call,
reported as the median and the range.  (a) and (b) compare their logp bit for bit, and (c) its samples.  The card's name, power
limit and SM clocks are read in the same process.  Prints one JSON object; --out DIR also writes DIR/score_model_bench.json.

    python tools/score_model_bench.py [--utterances 32] [--out DIR]
"""
import argparse
import json
import os
import statistics
import sys

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

S, A, MAXDIL = 256, 256, 512
ROWS, SAMPLES, CALLS, MODELS = 64, 4096, 5, 8
SHAPES = {"C3": (20, 64), "R128_L30": (30, 128)}


def timed(fn):
    """GPU seconds of fn() from CUDA events on the current stream, after a synchronise"""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3, out


def alternate(arms):
    """arms {name: fn}: a warm-up call of each, then CALLS rounds calling each once in turn.  Returns ({name: summary}, {name: last
    output})."""
    for fn in arms.values():
        fn()
    times, outs = {k: [] for k in arms}, {}
    for _ in range(CALLS):
        for k, fn in arms.items():
            t, outs[k] = timed(fn)
            times[k].append(t)
    return {k: {"median_ms": 1e3 * statistics.median(v), "min_ms": 1e3 * min(v), "max_ms": 1e3 * max(v)} for k, v in times.items()}, outs


def engine(w, L, R, B):
    e = nw.NVWavenetInfer(L, MAXDIL, B, SAMPLES, R=R, S=S, A=A, dtype=nw.FP16)
    e.load(w)
    return e


def scoring(name):
    L, R = SHAPES[name]
    ws = [refgen.lively_inputs(0x5C0 + m, R, S, A, L, 1, 1) for m in range(MODELS)]
    g = torch.Generator(device="cuda").manual_seed(11)
    lh = 0.5 * torch.randn((SAMPLES, L, ROWS, 2 * R), generator=g, device="cuda")
    audio = torch.randint(0, A, (ROWS, SAMPLES), dtype=torch.int32, device="cuda", generator=g)
    e = engine(ws[0], L, R, ROWS)
    for m in range(1, MODELS):
        d = engine(ws[m], L, R, 1)
        e.set_model(m, d)
        d.close()
    e.set_conditioning(lh, 0, SAMPLES)
    out = {"shape": {"L": L, "R": R, "S": S, "A": A, "max_dilation": MAXDIL, "rows": ROWS, "samples": SAMPLES}}
    for V in (2, 4, 8):
        table = [b % V for b in range(ROWS)]
        per = []                                                    # (b): V one-model engines of their own rows
        for m in range(V):
            rows = [b for b in range(ROWS) if table[b] == m]
            pe = engine(ws[m], L, R, len(rows))
            pe.set_conditioning(lh[:, :, rows].contiguous(), 0, SAMPLES)
            per.append((pe, rows, audio[rows].contiguous()))

        def mixed(tab):
            def run():
                e.set_score_models(tab)
                return e.score(audio)
            return run

        def separate():
            return [pe.score(a) for pe, _, a in per]

        res, outs = alternate({"zero_table": mixed([0] * ROWS), f"V{V}_table": mixed(table), f"V{V}_engines": separate})
        same = all(torch.equal(outs[f"V{V}_table"][rows].view(torch.int32), lp.view(torch.int32)) for (_, rows, _), lp in
                   zip(per, outs[f"V{V}_engines"]))
        res["bit_equal"] = bool(same)
        res["table_over_zero"] = res[f"V{V}_table"]["median_ms"] / res["zero_table"]["median_ms"]
        out[f"V{V}"] = res
        for pe, _, _ in per:
            pe.close()
    e.close()
    return out


def prompted(n):
    L, R = SHAPES["C3"]
    nets = [_net(refgen.lively_inputs(0x5C0 + m, R, S, A, L, 1, 1), L, R, S, A, MAXDIL) for m in range(4)]
    rng = np.random.default_rng(21)
    lengths = [int(v) for v in rng.integers(8000, 16001, n)]
    models = [int(v) for v in rng.integers(0, 4, n)]
    seeds = [int(v) for v in rng.integers(0, 2 ** 62, n)]
    prompts = [torch.from_numpy(rng.integers(0, A, int(rng.integers(1000, 4001))).astype(np.int32)).cuda() for _ in range(n)]
    g = torch.Generator(device="cuda").manual_seed(22)
    conds = [0.5 * torch.randn((2 * R, L, m), generator=g, device="cuda") for m in lengths]
    ms = ModelSet(nets)

    def together():
        return ms.infer_many(models, conds, seeds, slots=ROWS, window=SAMPLES, fp16=True, prompts=prompts)

    def apart():
        got = [None] * n
        for m, net in enumerate(nets):
            us = [u for u in range(n) if models[u] == m]
            if us:
                for u, o in zip(us, net.infer_many([conds[u] for u in us], [seeds[u] for u in us], slots=ROWS, window=SAMPLES, fp16=True,
                                                   prompts=[prompts[u] for u in us])):
                    got[u] = o
        return got

    res, outs = alternate({"modelset": together, "per_net": apart})
    res["bit_equal"] = all(torch.equal(a, b) for a, b in zip(outs["modelset"], outs["per_net"]))
    res["utterances"], res["samples"] = n, sum(lengths)
    ms.close()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--utterances", type=int, default=32)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("score_model_bench needs a CUDA device")
    result = {"card": card(), "calls_per_arm": CALLS}
    result["scoring"] = {name: scoring(name) for name in SHAPES}
    result["prompted_queue"] = prompted(args.utterances)
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "score_model_bench.json"), "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
