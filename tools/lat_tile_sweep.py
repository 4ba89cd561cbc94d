"""Both sides of the latency kernel's launch rule at the C3 model: for each batch, the kernel the rule picks (8-row clusters while
they are all resident, else 16-row clusters, else the single-CTA kernel) against the single-CTA kernel (NVWN_LAT_CLUSTER=0).
Kernel-only time, CUDA events, one warm-up run per engine.  python tools/lat_tile_sweep.py [B ...]   (default 64 128 256 384 512)"""
import json
import os
import subprocess
import sys

sys.path.insert(0, ".")
L, R, S, A, md = 20, 64, int(os.environ.get("S", 256)), 256, 512
N = int(os.environ.get("N", 4000))


def one(B, cluster):
    """One engine in this process: the switch is read at engine creation."""
    import numpy as np
    import torch
    import nv_wavenet_b200 as nw
    from tests import refgen
    os.environ["NVWN_FP16_KERNEL"] = "lat"
    os.environ["NVWN_LAT_CLUSTER"] = cluster
    w = refgen.lively_inputs(3, R, S, A, L, min(B, 16), 8)
    e = nw.NVWavenetInfer(L, md, B, N, R=R, S=S, A=A, dtype=nw.FP16)
    e.load(w)
    g = torch.Generator(device="cuda"); g.manual_seed(1)
    chunk = max(1, (64 << 20) // (L * B * 2 * R))
    for s0 in range(0, N, chunk):
        m = min(chunk, N - s0)
        e.set_conditioning((torch.rand((m, L, B, 2 * R), device="cuda", generator=g) - 0.5) * 0.5, s0, m)
    e.set_selectors(torch.rand((N, B), device="cuda", generator=g))
    torch.cuda.synchronize()
    y = torch.zeros((B, N), dtype=torch.int32, device="cuda")
    e.reset_history(); e.run(min(N, 200), B, None); torch.cuda.synchronize()
    e.reset_history()
    t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
    t0.record(); e.run(N, B, y); t1.record(); torch.cuda.synchronize()
    ms = t0.elapsed_time(t1)
    info = e.launch_info()
    crc = int(np.bitwise_xor.reduce(y.cpu().numpy().astype(np.uint32).ravel() * np.uint32(2654435761)))
    print(json.dumps({"B": B, "S": S, "N": N, "NVWN_LAT_CLUSTER": cluster, "cluster": info["cluster"], "batch_per_cta": info["batch_per_cta"],
                      "ms": round(ms, 3), "Msamples_s": round(B * N / ms / 1e3, 3), "yout_hash": f"{crc:08x}"}), flush=True)
    e.close()


if __name__ == "__main__":
    if len(sys.argv) == 4 and sys.argv[1] == "--one":
        one(int(sys.argv[2]), sys.argv[3])
        sys.exit(0)
    for B in [int(a) for a in sys.argv[1:]] or [64, 128, 256, 384, 512]:
        for cluster in ("1", "0"):
            subprocess.run([sys.executable, __file__, "--one", str(B), cluster], check=True)
