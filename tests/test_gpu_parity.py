"""GPU parity tests proper: the CUDA path, called through the C-ABI, against the CPU oracle.

fp32: bit-exact (indices AND every dumped activation) against oracle PORTABLE mode, which
test_oracle_pin.py pins to the reference CPU model; and exact indices against the golden vectors of
the reference's own nvWavenetReference on its 16 test runs (nv_wavenet_test.cu:343-394).
fp16: logits within 1e-2 relative (BASELINE.json north_star) at matched history (teacher forcing).
"""
import ctypes as C
import os

import numpy as np
import pytest

import nv_wavenet_b200 as nw
from oracle import pyoracle as po
from tests import common, refgen

pytestmark = pytest.mark.gpu

RUNS = common.reference_runs()


def gpu_engine(w, L, B, N, R, S, A, md, dtype=nw.FP32, tanh_embed=True, impl=nw.AUTO):
    e = nw.NVWavenetInfer(L, md, B, N, impl, tanh_embed, R=R, S=S, A=A, dtype=dtype)
    e.load(w)
    e.set_inputs(w["Lh"], w["selectors"])
    return e


def cpu_oracle(w, L, B, N, R, S, A, md, math=po.MATH_PORTABLE, prec=po.PREC_FP32, tanh_embed=True):
    o = po.Oracle(L, B, N, R, S, A, md, math=math, prec=prec, tanh_embed=tanh_embed)
    o.load(w)
    o.set_inputs(w["Lh"], w["selectors"])
    return o


def assert_acts_bit_equal(ao, ag):
    for k in ("xt", "skip", "zs", "za", "p"):
        assert common.bits_equal(ao[k], ag[k]), f"{k}: max abs diff {np.abs(ao[k] - ag[k]).max()}"


@pytest.mark.parametrize("run", RUNS, ids=[r[0] for r in RUNS])
def test_fp32_reference_test_runs(run):
    """The reference's own integration test, replayed: run_chunks(7, ...) twice, exact yOut, activations."""
    key, seed, i, R, S, A, L = run
    B, N, md = common.B_REF, common.N_REF, common.MAXDIL_REF
    w = common.reference_inputs(seed, i)
    g = common.golden()
    e = gpu_engine(w, L, B, N, R, S, A, md)
    o = cpu_oracle(w, L, B, N, R, S, A, md)
    for it in range(common.ITERS_REF):
        y = np.zeros((B, N), np.int32)
        seen = []
        assert e.run_chunks(7, lambda yo, init, n: seen.append((init, n)), N, B, y)
        e.synchronize()
        assert seen == [(0, 7), (7, 1)]
        yo = o.run(N, B)
        assert np.array_equal(y, g[key + "/y"][it]), "sampled indices differ from the reference CPU model"
        assert np.array_equal(y, yo)
        ag = e.activations()
        assert_acts_bit_equal(o.activations(), ag)
        # the reference test's own tolerances against its CPU model (nv_wavenet_test.cu:273-298)
        assert common.matrix_compare_ok(g[key + "/za"][it], ag["za"], 1e-4)
        assert common.matrix_compare_ok(g[key + "/p"][it], ag["p"], 1e-3)
        assert common.matrix_compare_ok(g[key + "/xt_last"][it], ag["xt"][-1], 1e-2)
        assert common.matrix_compare_ok(g[key + "/skip_last"][it], ag["skip"][-1], 1e-2, relu=True)


@pytest.mark.parametrize("shape", [
    # R, S, A, L, B, N, maxDil, BT
    (32, 128, 256, 5, 4, 40, 4, 1),
    (32, 128, 256, 5, 4, 40, 4, 4),
    (64, 128, 256, 4, 6, 24, 8, 2),
    (64, 256, 256, 6, 8, 70, 16, 4),      # ring wraps (N > maxDil+1) and dilation cycle restarts
    (64, 256, 256, 3, 3, 9, 2, 1),
    (128, 256, 256, 3, 4, 12, 4, 2),
    (64, 128, 512, 2, 2, 10, 2, 1),
    (128, 256, 1024, 2, 2, 6, 2, 2),
])
@pytest.mark.parametrize("gen", ["lively", "uniform"])
def test_fp32_bit_exact_fresh_shapes(shape, gen, monkeypatch):
    R, S, A, L, B, N, md, bt = shape
    monkeypatch.setenv("NVWN_STREAM_BT", str(bt))
    w = (refgen.lively_inputs if gen == "lively" else refgen.synthetic_inputs)(99 + R + N, R, S, A, L, B, N)
    e = gpu_engine(w, L, B, N, R, S, A, md)
    o = cpu_oracle(w, L, B, N, R, S, A, md)
    y = np.zeros((B, N), np.int32)
    assert e.run(N, B, y, dump_activations=True)
    e.synchronize()
    assert e.launch_info()["batch_per_cta"] == bt
    assert np.array_equal(y, o.run(N, B))
    assert_acts_bit_equal(o.activations(), e.activations())
    if gen == "lively":
        assert len(np.unique(y)) > 8          # a non-degenerate sampled distribution


def test_stream_switches_are_read_at_engine_creation(monkeypatch):
    """NVWN_STREAM_BT and NVWN_STREAM_RING hold for an engine from its creation on: changing them later does not reach its
    launches, and every new engine reads them again."""
    R, S, A, L, B, N, md = 64, 128, 256, 3, 4, 12, 4
    w = refgen.lively_inputs(8, R, S, A, L, B, N)
    monkeypatch.delenv("NVWN_STREAM_RING", raising=False)
    monkeypatch.setenv("NVWN_STREAM_BT", "4")
    e = gpu_engine(w, L, B, N, R, S, A, md)
    monkeypatch.setenv("NVWN_STREAM_BT", "1")
    assert e.run(N, B, np.zeros((B, N), np.int32)); e.synchronize()
    assert e.launch_info()["batch_per_cta"] == 4
    monkeypatch.delenv("NVWN_STREAM_BT")

    NT = max(4 * R, R + S, 128)                     # threads of the stream kernel; the weight ring adds one warp
    blocks, ys = [], []
    for ring in ("0", None):
        if ring is None:
            monkeypatch.delenv("NVWN_STREAM_RING")
        else:
            monkeypatch.setenv("NVWN_STREAM_RING", ring)
        e = gpu_engine(w, L, B, N, R, S, A, md)
        y = np.zeros((B, N), np.int32)
        assert e.run(N, B, y); e.synchronize()
        blocks.append(e.launch_info()["block"]); ys.append(y)
    assert blocks == [NT, NT + 32]
    assert np.array_equal(ys[0], ys[1])


def test_fp32_no_tanh_embed_and_forced_history():
    """tanhEmbed=false (the PyTorch export path, pytorch/wavenet.py:153-154) and teacher forcing."""
    R, S, A, L, B, N, md = 64, 256, 256, 4, 4, 20, 8
    w = refgen.lively_inputs(5, R, S, A, L, B, N)
    forced = np.random.default_rng(1).integers(0, A, (B, N)).astype(np.int32)
    e = gpu_engine(w, L, B, N, R, S, A, md, tanh_embed=False)
    o = cpu_oracle(w, L, B, N, R, S, A, md, tanh_embed=False)
    e.set_forced(forced); o.set_forced(forced)
    y = np.zeros((B, N), np.int32)
    e.run(N, B, y, dump_activations=True); e.synchronize()
    assert np.array_equal(y, o.run(N, B))
    assert_acts_bit_equal(o.activations(), e.activations())


_FAST_RUNS = list({r[3:6]: r for r in reversed(RUNS)}.values())          # the first reference run of every (R, S, A) shape


@pytest.mark.parametrize("run", _FAST_RUNS, ids=lambda r: r[0])
def test_fp32_fast_contract_on_reference_test_runs(run):
    """NVWN_FP32_FAST (FMA, two interleaved partial sums, float libm -- the arithmetic of the reference's GPU kernels): on the
    reference's own test runs the sampled indices equal the CPU model's and the activations stay within the reference test's own
    tolerances (nv_wavenet_test.cu:273-298), which is all the reference's kernels promise."""
    key, seed, i, R, S, A, L = run
    B, N, md = common.B_REF, common.N_REF, common.MAXDIL_REF
    w = common.reference_inputs(seed, i)
    g = common.golden()
    e = gpu_engine(w, L, B, N, R, S, A, md, dtype=nw.FP32_FAST)
    y = np.zeros((B, N), np.int32)
    e.run(N, B, y, dump_activations=True); e.synchronize()
    assert np.array_equal(y, g[key + "/y"][0]), "sampled indices differ from the reference CPU model"
    ag = e.activations()
    assert common.matrix_compare_ok(g[key + "/za"][0], ag["za"], 1e-4)
    assert common.matrix_compare_ok(g[key + "/p"][0], ag["p"], 1e-3)
    assert common.matrix_compare_ok(g[key + "/xt_last"][0], ag["xt"][-1], 1e-2)
    assert common.matrix_compare_ok(g[key + "/skip_last"][0], ag["skip"][-1], 1e-2, relu=True)


def test_fp32_fast_contract_lively_and_chunked():
    """Same contract on lively weights at the C4 shape (L30 R128 S256, maxDil 512): logits within 1e-4 of the bit-exact kernel at
    matched history, chunked == unchunked, and the free-running trajectories agree except where a selector sits on a boundary."""
    R, S, A, L, B, N, md = 128, 256, 256, 30, 4, 80, 512
    w = refgen.lively_inputs(17, R, S, A, L, B, N)
    ex = gpu_engine(w, L, B, N, R, S, A, md)
    ye = np.zeros((B, N), np.int32); ex.run(N, B, ye, dump_activations=True); ex.synchronize()
    fa = gpu_engine(w, L, B, N, R, S, A, md, dtype=nw.FP32_FAST)
    fa.set_forced(ye)
    yf = np.zeros((B, N), np.int32); fa.run(N, B, yf, dump_activations=True); fa.synchronize()
    za_e, za_f = ex.get_za(), fa.get_za()
    assert np.abs(za_f - za_e).max() <= 1e-4 * np.abs(za_e).max()
    assert (yf == ye).mean() > 0.99
    fa.set_forced(None); fa.reset_history()
    y1 = np.zeros((B, N), np.int32); fa.run(N, B, y1); fa.synchronize()
    fa.reset_history(); y2 = np.zeros((B, N), np.int32)
    fa.run_chunks(7, lambda *a: None, N, B, y2); fa.synchronize()
    assert np.array_equal(y1, y2)


def test_fp32_properties_at_full_model_size():
    """C3-sized model (L20 R64 S256 A256, maxDil 512), longer than the oracle can follow cheaply:
    chunked == unchunked, batch shards == whole batch, run-to-run determinism."""
    R, S, A, L, B, N, md = 64, 256, 256, 20, 8, 600, 512
    w = refgen.lively_inputs(11, R, S, A, L, B, N)
    e = gpu_engine(w, L, B, N, R, S, A, md)
    y1 = np.zeros((B, N), np.int32); e.run(N, B, y1); e.synchronize()
    # determinism
    e.reset_history(); y2 = np.zeros((B, N), np.int32); e.run(N, B, y2); e.synchronize()
    assert np.array_equal(y1, y2)
    # chunked
    e.reset_history(); y3 = np.zeros((B, N), np.int32)
    e.run_chunks(97, lambda *a: None, N, B, y3); e.synchronize()
    assert np.array_equal(y1, y3)
    # batch shards: utterances never interact (SURVEY.md §8e)
    for lo, hi in ((0, 4), (4, 8)):
        ws = dict(w); ws["Lh"] = np.ascontiguousarray(w["Lh"][:, :, lo:hi]); ws["selectors"] = np.ascontiguousarray(w["selectors"][:, lo:hi])
        es = gpu_engine(ws, L, hi - lo, N, R, S, A, md)
        ys = np.zeros((hi - lo, N), np.int32); es.run(N, hi - lo, ys); es.synchronize()
        assert np.array_equal(ys, y1[lo:hi])
    # oracle agrees on a prefix it can afford
    n0 = 48
    w0 = dict(w); w0["Lh"] = np.ascontiguousarray(w["Lh"][:n0]); w0["selectors"] = np.ascontiguousarray(w["selectors"][:n0])
    o = cpu_oracle(w0, L, B, n0, R, S, A, md)
    assert np.array_equal(o.run(n0, B), y1[:, :n0])


def test_fp32_device_pointers():
    """Weights / inputs / yOut given as device pointers (nv_wavenet_test.cu:133-239 variants)."""
    import torch
    R, S, A, L, B, N, md = 64, 128, 256, 3, 4, 10, 4
    w = refgen.lively_inputs(3, R, S, A, L, B, N)
    wd = {k: torch.from_numpy(v).cuda() for k, v in w.items()}
    e = nw.NVWavenetInfer(L, md, B, N, R=R, S=S, A=A)
    e.load(wd); e.set_inputs(wd["Lh"], wd["selectors"])
    yd = torch.zeros((B, N), dtype=torch.int32, device="cuda")
    e.run(N, B, yd, dump_activations=True); e.synchronize()
    o = cpu_oracle(w, L, B, N, R, S, A, md)
    assert np.array_equal(yd.cpu().numpy(), o.run(N, B))


def _logit_check(za_o, za_g, rel=1e-2, mean_rel=None):
    """BASELINE.json north_star: fp16 logits within 1e-2 relative.  A logit that cancels to ~0 has no meaningful
    relative error, so each one is judged against max(|z|, 0.25 * max|z| of its utterance)."""
    scale = np.abs(za_o).max(axis=-1, keepdims=True)
    err = np.abs(za_g - za_o)
    assert np.all(err <= rel * np.maximum(np.abs(za_o), 0.25 * scale)), f"max err / scale {(err / scale).max()}"
    if mean_rel is not None:
        assert (err / scale).mean() <= mean_rel, f"mean err / scale {(err / scale).mean()}"


FP16_KERNELS = ["stream", "lat", "lat_single", "tc", "tc_tile32_fused", "tc_tile64_fused", "tc_nodup"]


def _select_fp16_kernel(kernel, monkeypatch):
    """Environment switches read once by nvwn_create: which fp16 kernel, and which tile shape / schedule of the tensor-core one."""
    for k in ("NVWN_FP16_KERNEL", "NVWN_TC_TILE", "NVWN_TC_NODUP", "NVWN_TC_FUSED", "NVWN_LAT_CLUSTER"):
        monkeypatch.delenv(k, raising=False)
    if kernel == "stream":
        monkeypatch.setenv("NVWN_FP16_KERNEL", "stream")
    elif kernel == "lat":                          # latency-mode kernel (mma.sync, 16-utterance tiles, a three-CTA cluster per tile while all clusters are resident): AUTO
        monkeypatch.setenv("NVWN_FP16_KERNEL", "lat")
    elif kernel == "lat_single":                   # ... one CTA per tile: what AUTO uses once the clusters no longer fit one wave
        monkeypatch.setenv("NVWN_FP16_KERNEL", "lat"); monkeypatch.setenv("NVWN_LAT_CLUSTER", "0")
    else:                                          # tensor-core (wgmma) kernel; "tc" = the default 64-utterance tiles, unfused schedule
        monkeypatch.setenv("NVWN_FP16_KERNEL", "tc")
        if kernel == "tc_nodup":                   # 128-utterance tiles, two CTAs per tile (see resolve_config in wn_engine.cu)
            monkeypatch.setenv("NVWN_TC_NODUP", "1")
        if kernel == "tc_tile32_fused":            # 32-utterance tiles run the fused schedule
            monkeypatch.setenv("NVWN_TC_TILE", "32")
        if kernel == "tc_tile64_fused":            # fused schedule on 64-utterance tiles
            monkeypatch.setenv("NVWN_TC_TILE", "64"); monkeypatch.setenv("NVWN_TC_FUSED", "1")


def _check_sampled_index(p, sel, y):
    """y must be the first class whose cumulative probability exceeds the selector (reference.cpp:106-121), judged on the
    kernel's own dumped p; a selector within 1e-4 of a boundary may fall on either side."""
    cs = np.cumsum(p.astype(np.float64), axis=1)
    cs /= cs[:, -1:]
    for b in range(p.shape[0]):
        lo = int(np.searchsorted(cs[b], sel[b] - 1e-4, side="right"))
        hi = int(np.searchsorted(cs[b], sel[b] + 1e-4, side="right"))
        assert lo <= y[b] <= min(hi, p.shape[1] - 1), f"utterance {b}: sampled {y[b]}, expected [{lo}, {hi}] for selector {sel[b]}"


@pytest.mark.parametrize("kernel", FP16_KERNELS)
@pytest.mark.parametrize("shape", [
    (64, 256, 256, 20, 8, 24, 8),
    (64, 128, 256, 20, 4, 16, 4),
    (64, 256, 256, 20, 64, 12, 4),
    (64, 256, 256, 20, 130, 6, 2),        # several batch tiles, the last one nearly empty
    (64, 256, 256, 5, 100, 10, 16),       # odd layer count, partially filled tile
    (64, 256, 256, 12, 20, 30, 4),        # the shortest stack the cluster kernel takes
    (64, 256, 256, 16, 20, 24, 128, False),   # the exported model's configuration (refgen.export_inputs): no embedding tanh
])
def test_fp16_logits_teacher_forced(shape, kernel, monkeypatch):
    R, S, A, L, B, N, md, tanh_embed = shape + (True,) * (8 - len(shape))
    _select_fp16_kernel(kernel, monkeypatch)
    w = (refgen.lively_inputs if tanh_embed else refgen.export_inputs)(21 + B, R, S, A, L, B, N)
    o32 = cpu_oracle(w, L, B, N, R, S, A, md, tanh_embed=tanh_embed)
    forced = o32.run(N, B)                                     # the fp32 model's own trajectory as history
    for n_run in (1, N):                                       # step 0 (identical history) and the last step
        wn_ = dict(w); wn_["Lh"] = np.ascontiguousarray(w["Lh"][:n_run]); wn_["selectors"] = np.ascontiguousarray(w["selectors"][:n_run])
        f = np.ascontiguousarray(forced[:, :n_run])
        e = gpu_engine(wn_, L, B, n_run, R, S, A, md, dtype=nw.FP16, tanh_embed=tanh_embed)
        e.set_forced(f)
        y = np.zeros((B, n_run), np.int32)
        e.run(n_run, B, y, dump_activations=True); e.synchronize()
        assert e.launch_info()["kernel"] == {"stream": 16, "lat": 18, "lat_single": 18}.get(kernel, 17)
        if kernel.startswith("lat"):
            assert e.launch_info()["cluster"] == (3 if kernel == "lat" and L >= 12 else 1)     # shorter stacks: single-CTA kernel
        o16 = cpu_oracle(wn_, L, B, n_run, R, S, A, md, prec=po.PREC_FP16, tanh_embed=tanh_embed); o16.set_forced(f); o16.run(n_run, B)
        o = cpu_oracle(wn_, L, B, n_run, R, S, A, md, tanh_embed=tanh_embed); o.set_forced(f); o.run(n_run, B)
        ag = e.activations()
        _logit_check(o16.get_za(), ag["za"], 1e-2, mean_rel=3e-4)   # vs the fp16-contract oracle (catches layout slips)
        _logit_check(o.get_za(), ag["za"], 1e-2)                    # vs the fp32 oracle: the north-star tolerance
        assert np.allclose(ag["p"].sum(axis=1), 1.0, atol=1e-3)
        assert np.abs(ag["p"] - o.get_p()).max() <= 1e-2 * o.get_p().max()
        _check_sampled_index(ag["p"], wn_["selectors"][n_run - 1], y[:, n_run - 1])
        if kernel.startswith("lat"):
            # intermediate activations of the last step against the fp16-contract oracle
            ao = o16.activations()
            for k, tol in (("xt", 2e-2), ("skip", 2e-2), ("zs", 2e-2)):
                sc = np.abs(ao[k]).max()
                assert np.abs(ag[k] - ao[k]).max() <= tol * sc, f"{k}: {np.abs(ag[k] - ao[k]).max() / sc}"


@pytest.mark.parametrize("shape", [
    (32, 128, 256, 6, 5, 14, 4),          # R32: reference shape (README.md:7-10); the mma kernels are R64-only
    (128, 256, 256, 4, 3, 10, 4),         # R128
    (64, 128, 512, 4, 3, 10, 2),          # A = 512 (nv_wavenet_test.cu:391-394)
    (64, 256, 256, 3, 4, 12, 4),          # L < 4: below the latency kernel's prefetch depth
])
def test_fp16_fallback_shapes_use_the_stream_kernel(shape, monkeypatch):
    """fp16 on shapes outside the tensor-core kernels' set: AUTO must fall back to the CUDA-core stream kernel (no error, no other
    path), and its logits must meet the same fp16 tolerance against the oracle."""
    for k in ("NVWN_FP16_KERNEL", "NVWN_TC_TILE", "NVWN_TC_NODUP", "NVWN_TC_FUSED"):
        monkeypatch.delenv(k, raising=False)
    R, S, A, L, B, N, md = shape
    w = refgen.lively_inputs(40 + R + A, R, S, A, L, B, N)
    o = cpu_oracle(w, L, B, N, R, S, A, md)
    forced = o.run(N, B)
    e = gpu_engine(w, L, B, N, R, S, A, md, dtype=nw.FP16)
    e.set_forced(forced)
    y = np.zeros((B, N), np.int32)
    e.run(N, B, y, dump_activations=True); e.synchronize()
    expect = 17 if (R, A) == (64, 256) and L < 4 else 16          # R64/A256 with L < 4: the tensor-core kernel still applies
    assert e.launch_info()["kernel"] == expect
    o16 = cpu_oracle(w, L, B, N, R, S, A, md, prec=po.PREC_FP16); o16.set_forced(forced); o16.run(N, B)
    ag = e.activations()
    _logit_check(o16.get_za(), ag["za"], 1e-2, mean_rel=3e-4)
    _logit_check(o.get_za(), ag["za"], 1e-2)
    _check_sampled_index(ag["p"], w["selectors"][N - 1], y[:, N - 1])


def _run_range(e, init, count, N, B, y=None):
    """run_partial over samples [init, init+count) of an N-sample batch (the reference's run_partial + samples_per_chunk)."""
    e._samples_per_chunk = count
    e.run_partial(init, N, B, y)
    e._samples_per_chunk = 0


@pytest.mark.parametrize("kernel", ["lat", "lat_single", "tc"])      # "tc" = the tensor-core kernel's default: 64-utterance tiles, unfused schedule
def test_fp16_soak_determinism_and_chunking(kernel, monkeypatch):
    """The fp16 kernels at the C3 shape (L20 R64 S256 A256, maxDil 512, 64 utterances) over 2000 samples -- several turns of the
    513-slot history ring and of the dilation cycle: run twice -> identical yOut; run_chunks(97) and three unequal
    run_partial pieces == one launch, bit for bit (reference: nv_wavenet_test.cu:254,302-304 chunks of 7+1, exact indices)."""
    R, S, A, L, B, N, md = 64, 256, 256, 20, 64, 2000, 512
    _select_fp16_kernel(kernel, monkeypatch)
    w = refgen.lively_inputs(31, R, S, A, L, B, N)
    e = gpu_engine(w, L, B, N, R, S, A, md, dtype=nw.FP16)
    y1 = np.zeros((B, N), np.int32); e.run(N, B, y1); e.synchronize()
    assert len(np.unique(y1)) > 32
    for _ in range(3):
        e.reset_history(); y2 = np.zeros((B, N), np.int32); e.run(N, B, y2); e.synchronize()
        assert np.array_equal(y1, y2), "run-to-run determinism"
    e.reset_history(); y3 = np.zeros((B, N), np.int32)
    seen = []
    e.run_chunks(97, lambda yo, init, n: seen.append((init, n)), N, B, y3); e.synchronize()
    assert seen[0] == (0, 97) and seen[-1] == (1940, 60)
    assert np.array_equal(y1, y3), "run_chunks(97) != one launch"
    e.reset_history(); y4 = np.zeros((B, N), np.int32)
    _run_range(e, 0, 1, N, B); _run_range(e, 1, 700, N, B); _run_range(e, 701, 1299, N, B, y4); e.synchronize()
    assert np.array_equal(y1, y4), "three unequal run_partial pieces != one launch"


@pytest.mark.parametrize("kernel", ["lat", "lat_single", "tc"])
def test_fp16_logits_after_ring_wrap(kernel, monkeypatch):
    """Teacher-forced logits at step N-1 = 599 > maxDil + 1 = 513 (real ring wrap, every dilation live) against the oracle."""
    R, S, A, L, B, N, md = 64, 256, 256, 20, 16, 600, 512
    _select_fp16_kernel(kernel, monkeypatch)
    w = refgen.lively_inputs(57, R, S, A, L, B, N)
    forced = np.random.default_rng(5).integers(0, A, (B, N)).astype(np.int32)
    e = gpu_engine(w, L, B, N, R, S, A, md, dtype=nw.FP16)
    e.set_forced(forced)
    y = np.zeros((B, N), np.int32)
    e.run(N, B, y, dump_activations=True); e.synchronize()
    o = cpu_oracle(w, L, B, N, R, S, A, md); o.set_forced(forced); o.run(N, B)
    ag = e.activations()
    _logit_check(o.get_za(), ag["za"], 1e-2)
    _check_sampled_index(ag["p"], w["selectors"][N - 1], y[:, N - 1])


def test_fp16_latency_kernel_smaller_batch_than_engine():
    """run(batch_size < engine batch): the first batch_size utterances of the engine's batch (16-utterance tiles are independent)."""
    R, S, A, L, B, N, md = 64, 256, 256, 6, 40, 30, 8
    w = refgen.lively_inputs(8, R, S, A, L, B, N)
    e = gpu_engine(w, L, B, N, R, S, A, md, dtype=nw.FP16, impl=nw.KERNEL_LATENCY)
    y_all = np.zeros((B, N), np.int32); e.run(N, B, y_all); e.synchronize()
    e.reset_history()
    # selectors are indexed with the run's batch size as the stride (nv_wavenet.cuh:144): [N][20] at the front of the buffer
    e.set_selectors(np.concatenate([np.ascontiguousarray(w["selectors"][:, :20]).reshape(-1), np.zeros(N * (B - 20), np.float32)]))
    y20 = np.zeros((20, N), np.int32); e.run(N, 20, y20); e.synchronize()
    assert np.array_equal(y20, y_all[:20])


def test_wavenet_infer_c_abi_drop_in():
    """The reference C-ABI entry point (pytorch/wavenet_infer.h:28-58): float** layer arrays, selectors
    from libc rand() -- seeded here so the expected draw can be replayed -- zero output biases."""
    from nv_wavenet_b200 import _lib
    lib = _lib.lib()
    R, S, A = lib.get_R(), lib.get_S(), lib.get_A()
    L, B, N, md = 4, 4, 16, 4
    w = refgen.lively_inputs(77, R, S, A, L, B, N)
    libc = C.CDLL(None)
    libc.srand(1234)
    arr = lambda key: (C.c_void_p * L)(*[w[key][l].ctypes.data for l in range(L)])
    samples = np.zeros((B, N), np.int32)
    lib.wavenet_infer(N, B, w["embPrev"].ctypes.data, w["embCur"].ctypes.data, L, md,
                      arr("Wprev"), arr("Wcur"), arr("Bh"), arr("Wres"), arr("Bres"), arr("Wskip"), arr("Bskip"),
                      w["Wzs"].ctypes.data, w["Wza"].ctypes.data, 1, w["Lh"].ctypes.data, 3, samples.ctypes.data)
    # expected selectors: Matrix(batch, samples).randomize(0.5, 1.0) on the same rand() stream
    rng = refgen.GlibcRand(1234)
    sel = refgen.randomize(rng, B, N, np.float32(0.5), np.float32(1.0)).reshape(N, B)
    w2 = dict(w); w2["selectors"] = sel; w2["Bzs"] = np.zeros(A, np.float32); w2["Bza"] = np.zeros(A, np.float32)
    o = cpu_oracle(w2, L, B, N, R, S, A, md)
    assert np.array_equal(samples, o.run(N, B))


def test_nvwavenet_python_class_matches_oracle():
    """pytorch/nv_wavenet.py surface (NVWaveNet(**export_weights()).infer(cond_input, impl)): conv-style weight shapes,
    one extra (unused) residual layer appended, cond_input channels x batch x layers x samples; device tensors."""
    import torch
    from nv_wavenet_b200.nv_wavenet import Impl, NVWaveNet
    R, S, A, L, B, N, md = 64, 256, 256, 3, 2, 12, 4
    w = refgen.lively_inputs(123, R, S, A, L, B, N)
    dev = "cuda"
    tt = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    cm = lambda flat, M, K: np.ascontiguousarray(flat.reshape(K, M).T)             # column-major flat -> row-major [M][K]
    dilate = [tt(np.stack([cm(w["Wprev"][l], 2 * R, R), cm(w["Wcur"][l], 2 * R, R)], axis=2)) for l in range(L)]
    net = NVWaveNet(embedding_prev=tt(w["embPrev"]), embedding_curr=tt(w["embCur"]),
                    conv_out_weight=tt(cm(w["Wzs"], A, S)[:, :, None]), conv_end_weight=tt(cm(w["Wza"], A, A)[:, :, None]),
                    dilate_weights=dilate, dilate_biases=[tt(w["Bh"][l]) for l in range(L)], max_dilation=md,
                    res_weights=[tt(cm(w["Wres"][l], R, R)[:, :, None]) for l in range(L - 1)],
                    res_biases=[tt(w["Bres"][l]) for l in range(L - 1)],
                    skip_weights=[tt(cm(w["Wskip"][l], S, R)[:, :, None]) for l in range(L)],
                    skip_biases=[tt(w["Bskip"][l]) for l in range(L)], use_embed_tanh=True)
    cond = tt(np.ascontiguousarray(w["Lh"].transpose(3, 2, 1, 0)))               # [2R][B][L][N]
    C.CDLL(None).srand(99)
    y = net.infer(cond, Impl.PERSISTENT).cpu().numpy()
    rng = refgen.GlibcRand(99)
    w2 = dict(w)
    w2["selectors"] = refgen.randomize(rng, B, N, np.float32(0.5), np.float32(1.0)).reshape(N, B)
    w2["Bzs"] = np.zeros(A, np.float32); w2["Bza"] = np.zeros(A, np.float32)
    w2["Wres"] = w["Wres"].copy(); w2["Bres"] = w["Bres"].copy()
    w2["Wres"][L - 1] = 0; w2["Bres"][L - 1] = 0                                # the appended, unused last residual layer
    o = cpu_oracle(w2, L, B, N, R, S, A, md)
    assert np.array_equal(y, o.run(N, B))
