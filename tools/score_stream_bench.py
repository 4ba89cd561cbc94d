"""Streaming scoring (nvwn_score_stream) through NVWaveNet: windowed against whole-length log-likelihood, and long audio from mel
frames through a fixed-size engine.

    python tools/score_stream_bench.py --out DIR [--calls 5] [--warmup 1]

C3 model (R64 / S256 / A256, 20 layers, max dilation 512, fp16) with lively seeded weights, seeded audio and seeded mel frames (80
channels, upsampling window 800, stride 200).  Two arms, their calls alternated round by round after `warmup` rounds, each call
timed with CUDA events and ending in a device synchronise (as the calls themselves do):
  a  64 x 16 000 samples: NVWaveNet.log_likelihood of the whole length against window=4000, from the same fp32 conditioning;
     ms per call, samples/s, and whether logp is bit-equal between the two.
  b  64 x 160 000 samples from frames: log_likelihood_from_features(window=16000); ms per call, samples/s, the device bytes of the
     engine and its scratch (free device memory before and after the first call, less what torch's allocator took), the split
     between production and scoring, and the bytes the whole-length path would need, computed from shapes and not run.
The card's name, power limit and max SM clock come from the read-only nvidia-smi query of tools/score_bench.py.  Writes
DIR/score_stream_bench.json and prints it.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nv_wavenet_b200.nv_wavenet import NVWaveNet  # noqa: E402
from tools.score_bench import card  # noqa: E402

R, S, A, L, MD = 64, 256, 256, 20, 512
B = 64
C_MEL, K_MEL, STRIDE = 80, 800, 200
A_SAMPLES, A_WINDOW = 16000, 4000
B_SAMPLES, B_WINDOW = 160000, 16000


def c3_net(seed):
    """NVWaveNet of the C3 shape with O(1) gates and logits far from uniform (the scales of tests/refgen.py lively_inputs)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = lambda *shape, s: s * torch.randn(shape, generator=g, device="cuda")
    return NVWaveNet(embedding_prev=n(A, R, s=0.7), embedding_curr=n(A, R, s=0.7), conv_out_weight=n(A, S, s=1 / np.sqrt(S)),
                     conv_end_weight=n(A, A, s=2 / np.sqrt(A)), dilate_weights=[n(2 * R, R, 2, s=0.7 / np.sqrt(R)) for _ in range(L)],
                     dilate_biases=[n(2 * R, s=0.1) for _ in range(L)], max_dilation=MD,
                     res_weights=[n(R, R, s=0.5 / np.sqrt(R)) for _ in range(L - 1)], res_biases=[n(R, s=0.05) for _ in range(L - 1)],
                     skip_weights=[n(S, R, s=0.5 / np.sqrt(R)) for _ in range(L)], skip_biases=[n(S, s=0.05) for _ in range(L)],
                     use_embed_tanh=True)


def timed_call(fn):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    out = fn()
    ev[1].record()
    torch.cuda.synchronize()
    return out, ev[0].elapsed_time(ev[1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("score_stream_bench needs a CUDA device")
    calls = max(a.calls, 5)
    net = c3_net(41)
    g = torch.Generator(device="cuda").manual_seed(42)

    # arm a: expanded fp32 conditioning, channels x batch x num_layers x samples
    cond = 0.5 * torch.randn((2 * R, B, L, A_SAMPLES), generator=g, device="cuda")
    audio_a = torch.randint(0, A, (B, A_SAMPLES), generator=g, device="cuda", dtype=torch.int32)
    whole = lambda: net.log_likelihood(cond, audio_a)
    windowed = lambda: net.log_likelihood(cond, audio_a, window=A_WINDOW)

    # arm b: mel frames and the conditioning network
    frames = B_SAMPLES // STRIDE
    features = torch.randn((B, C_MEL, frames), generator=g, device="cuda")
    cnet = (torch.randn((C_MEL, C_MEL, K_MEL), generator=g, device="cuda") / np.sqrt(C_MEL * K_MEL / STRIDE),
            0.1 * torch.randn(C_MEL, generator=g, device="cuda"),
            0.5 * torch.randn((L * 2 * R, C_MEL), generator=g, device="cuda") / np.sqrt(C_MEL),
            0.1 * torch.randn(L * 2 * R, generator=g, device="cuda"))
    audio_b = torch.randint(0, A, (B, B_SAMPLES), generator=g, device="cuda", dtype=torch.int32)
    split = {}
    from_frames = lambda: net.log_likelihood_from_features(features, audio_b, *cnet, STRIDE, window=B_WINDOW, timing=split)

    torch.cuda.synchronize()
    free0, reserved0 = torch.cuda.mem_get_info()[0], torch.cuda.memory_reserved()
    from_frames()
    free1, reserved1 = torch.cuda.mem_get_info()[0], torch.cuda.memory_reserved()
    engine_bytes = (free0 - free1) - (reserved1 - reserved0)

    for _ in range(a.warmup):
        whole(); windowed(); from_frames()
    ms = {"whole": [], "window": [], "frames": []}
    produce_ms, score_ms = [], []
    equal = True
    for _ in range(calls):
        lp_whole, t = timed_call(whole)
        ms["whole"].append(t)
        lp_window, t = timed_call(windowed)
        ms["window"].append(t)
        equal = equal and torch.equal(lp_whole.view(torch.int32), lp_window.view(torch.int32))
        lp_frames, t = timed_call(from_frames)
        ms["frames"].append(t)
        produce_ms.append(split["produce_s"] * 1e3)
        score_ms.append(split["score_s"] * 1e3)
        del lp_whole, lp_window

    med = {k: float(np.median(v)) for k, v in ms.items()}
    n_a, n_b = B * A_SAMPLES, B * B_SAMPLES
    store_per_sample = L * ((B + 15) // 16) * 4096                  # the latency engines' fp16 store: 16-utterance tiles of [L][2R]
    res = {
        "card": card(),
        "model": {"R": R, "S": S, "A": A, "L": L, "max_dilation": MD, "dtype": "fp16"},
        "calls": calls, "warmup": a.warmup,
        "arm_a": {"batch": B, "samples": A_SAMPLES, "window": A_WINDOW,
                  "whole_ms": ms["whole"], "whole_ms_median": med["whole"], "whole_samples_per_s": n_a / (med["whole"] * 1e-3),
                  "window_ms": ms["window"], "window_ms_median": med["window"], "window_samples_per_s": n_a / (med["window"] * 1e-3),
                  "window_over_whole": med["window"] / med["whole"], "logp_bit_equal": bool(equal)},
        "arm_b": {"batch": B, "samples": B_SAMPLES, "window": B_WINDOW, "mel_channels": C_MEL, "upsample_window": K_MEL, "stride": STRIDE,
                  "ms": ms["frames"], "ms_median": med["frames"], "samples_per_s": n_b / (med["frames"] * 1e-3),
                  "produce_ms": produce_ms, "produce_ms_median": float(np.median(produce_ms)),
                  "score_ms": score_ms, "score_ms_median": float(np.median(score_ms)),
                  "engine_and_scratch_bytes": int(engine_bytes),
                  "mean_neg_logp": float(-lp_frames.double().mean().item()),
                  "not_run_whole_length_store_bytes": B_SAMPLES * store_per_sample,
                  "not_run_whole_length_fp32_conditioning_bytes": n_b * L * 2 * R * 4,
                  "frames_bytes": B * C_MEL * frames * 4},
    }
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "score_stream_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
