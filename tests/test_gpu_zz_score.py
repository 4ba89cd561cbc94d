"""Teacher-forced scoring (nvwn_score): per-sample log-likelihood of given audio, every step at once.

Checked against the CPU oracle's logit trace at every step, against the dumped logits of forced generation, across the
three engine kinds, for bit-exact determinism and causality, and for leaving the generation state alone."""
import ctypes as C

import numpy as np
import pytest
import torch

import nv_wavenet_b200 as nw
from nv_wavenet_b200 import _lib
from oracle import pyoracle as po
from tests import common, refgen, replay

pytestmark = pytest.mark.gpu

EINVAL, EUNSUPPORTED = -1, -2
KINDS = {"lat": nw.KERNEL_LATENCY, "tc": nw.KERNEL_TENSORCORE, "stream": nw.KERNEL_STREAM}


def _fp16_rule(z_ref, z, mean_rel=None):
    scale = np.abs(z_ref).max(axis=-1, keepdims=True)
    err = np.abs(z - z_ref)
    assert np.all(err <= 1e-2 * np.maximum(np.abs(z_ref), 0.25 * scale)), f"max err / scale {(err / scale).max()}"
    if mean_rel is not None:
        assert (err / scale).mean() <= mean_rel, f"mean err / scale {(err / scale).mean()}"


def _log_softmax64(z):
    z = np.asarray(z, np.float64)
    mx = z.max(axis=-1, keepdims=True)
    lse = mx + np.log(np.exp(z - mx).sum(axis=-1, keepdims=True))
    return z - lse, lse[..., 0]


def _engine(w, L, B, N, R, S, A, md, impl=nw.AUTO, tanh_embed=True):
    e = nw.NVWavenetInfer(L, md, B, N, impl, tanh_embed, R=R, S=S, A=A, dtype=nw.FP16)
    e.load(w)
    e.set_inputs(w["Lh"], w["selectors"])
    return e


@pytest.mark.parametrize("shape", [
    (32, 128, 256, 20, 4, 24, 8, True),
    (64, 128, 256, 20, 4, 24, 8, True),
    (64, 256, 256, 20, 4, 24, 8, True),
    (128, 256, 256, 30, 3, 16, 8, True),
    (64, 256, 256, 4, 64, 800, 512, True),        # 256-step chunks at B = 64: the second chunk boundary is 544 steps in
    (64, 256, 256, 20, 4, 24, 8, False),          # the export path: no embedding tanh, zero embPrev
    (64, 256, 256, 16, 72, 160, 128, "export"),   # the exported model's configuration (refgen.export_inputs) at L16 maxDil 128
])
def test_oracle_parity_at_every_step(shape):
    R, S, A, L, B, N, md, tanh_embed = shape
    if tanh_embed == "export":
        tanh_embed = False
        w = refgen.export_inputs(70 + L + R, R, S, A, L, B, N)
    else:
        w = refgen.lively_inputs(70 + L + R, R, S, A, L, B, N)
    if not tanh_embed:
        w["embPrev"] = np.zeros_like(w["embPrev"])
    # utterances the CPU oracle follows (rows are independent): the scorer's rows t * B + b run in 64-row tiles, so at B >= 64
    # rows sit at both edges of a tile's 8- and 16-row groups, at the tile's middle and end, and in the ragged last tile
    rows = [b for b in (0, 7, 8, 31, 32, 56, 63, 64, 71) if b < B] if B >= 64 else list(range(min(B, 8)))
    Bo = len(rows)
    audio, z32 = replay.oracle_trace(w, rows, (R, S, A, L, md), N, tanh_embed=tanh_embed)      # the fp32 model's own trajectory
    _, z16 = replay.oracle_trace(w, rows, (R, S, A, L, md), N, forced=audio, tanh_embed=tanh_embed, prec=po.PREC_FP16)
    full_audio = np.random.default_rng(1).integers(0, A, (B, N)).astype(np.int32)
    full_audio[rows] = audio
    e = _engine(w, L, B, N, R, S, A, md, tanh_embed=tanh_embed)
    logp, logits = e.score(full_audio, logits=True)
    logp, logits = logp[rows], logits[rows]
    assert logits.shape == (Bo, N, A) and np.isfinite(logits).all()
    _fp16_rule(z16, logits, mean_rel=3e-4)                            # the fp16 contract
    _fp16_rule(z32, logits)                                           # the fp32 model
    ls32, _ = _log_softmax64(z32)
    want = np.take_along_axis(ls32, audio[..., None].astype(np.int64), -1)[..., 0]
    assert np.all(np.abs(logp - want) <= 2e-2 * np.abs(z32).max(axis=-1))
    own, lse = _log_softmax64(logits)
    own = np.take_along_axis(own, audio[..., None].astype(np.int64), -1)[..., 0]
    assert np.all(np.abs(logp - own) <= 1e-5 * (1 + np.abs(lse)))


def test_engine_kinds_agree_with_generation_and_each_other():
    R, S, A, L, B, N, md = 64, 256, 256, 20, 64, 40, 16
    w = refgen.lively_inputs(5, R, S, A, L, B, N)
    audio = np.random.default_rng(2).integers(0, A, (B, N)).astype(np.int32)
    ref = None
    for kind, impl in KINDS.items():
        e = _engine(w, L, B, N, R, S, A, md, impl=impl)
        logp, logits = e.score(audio, logits=True)
        e.set_forced(audio)
        y = np.zeros((B, N), np.int32)
        e.run(N, B, y, dump_activations=True)
        e.synchronize()
        assert e.launch_info()["kernel"] == {"lat": 18, "tc": 17, "stream": 16}[kind]
        _fp16_rule(e.get_za(), logits[:, N - 1])
        if ref is None:
            ref = logp
        else:
            assert common.bits_equal(ref, logp), f"{kind}: logp differs from the latency engine's"


def _c3_engine(B, N, seed=3, of=None):
    """C3 model with random conditioning for the first B of `of` (default B) utterances."""
    R, S, A, L, md = 64, 256, 256, 20, 512
    w = refgen.lively_inputs(seed, R, S, A, L, 1, 1)
    g = torch.Generator(device="cuda").manual_seed(seed)
    lh = 0.5 * torch.randn((N, L, of or B, 2 * R), generator=g, device="cuda")
    lh = lh[:, :, :B].contiguous()
    e = nw.NVWavenetInfer(L, md, B, N, R=R, S=S, A=A, dtype=nw.FP16)
    e.load(w)
    e.set_conditioning(lh, 0, N)
    torch.cuda.synchronize()
    return e


def test_determinism_and_causality_at_c3():
    B, N = 64, 3 * 256 + 100                                          # four chunks of 256 steps at B = 64
    e = _c3_engine(B, N)
    audio = np.random.default_rng(4).integers(0, 256, (B, N)).astype(np.int32)
    a = e.score(audio)
    assert np.isfinite(a).all() and (a <= 0).all()
    assert common.bits_equal(a, e.score(audio)), "a repeated call differs"
    n = 300
    assert common.bits_equal(a[:, :n], e.score(audio, num_samples=n)), "num_samples changes the bits"
    t0 = 400
    changed = audio.copy()
    changed[:, t0 + 1:] = np.random.default_rng(5).integers(0, 256, (B, N - t0 - 1))
    assert common.bits_equal(a[:, :t0 + 1], e.score(changed)[:, :t0 + 1]), "a later sample changed an earlier logp"
    assert common.bits_equal(a[:5], e.score(audio, batch_size=5)), "batch_size changes the bits"
    e5 = _c3_engine(5, N, of=B)
    assert common.bits_equal(a[:5], e5.score(audio[:5])), "an engine on a slice of the utterances differs"


def test_generation_state_untouched():
    R, S, A, L, B, N, md, n1 = 64, 256, 256, 12, 16, 30, 8, 11
    w = refgen.lively_inputs(6, R, S, A, L, B, N)
    one = _engine(w, L, B, N, R, S, A, md)
    y1 = np.zeros((B, N), np.int32)
    one.run(N, B, y1, dump_activations=True); one.synchronize()
    e = _engine(w, L, B, N, R, S, A, md)
    y = np.zeros((B, N), np.int32)
    lib = _lib.lib()
    _lib.check(lib.nvwn_run_partial(e._h, 0, n1, N, B, None, 1, None), "run_partial")
    e.synchronize()
    acts, info = e.activations(), e.launch_info()
    e.score(np.random.default_rng(7).integers(0, A, (B, N)).astype(np.int32), logits=True)
    after = e.activations()
    for k in acts:
        assert common.bits_equal(acts[k], after[k]), f"score changed the {k} dump"
    assert e.launch_info() == info, "score changed the launch info"
    _lib.check(lib.nvwn_run_partial(e._h, n1, N - n1, N, B, C.c_void_p(y.ctypes.data), 1, None), "run_partial")
    e.synchronize()
    assert np.array_equal(y, y1)
    a1, a2 = one.activations(), e.activations()
    for k in a1:
        assert common.bits_equal(a1[k], a2[k]), k


def test_weight_updates_reach_the_scorer():
    R, S, A, L, B, N, md = 64, 256, 256, 12, 8, 40, 8
    w = refgen.lively_inputs(8, R, S, A, L, B, N)
    w2 = refgen.lively_inputs(9, R, S, A, L, B, N)
    audio = np.random.default_rng(9).integers(0, A, (B, N)).astype(np.int32)
    e = _engine(w, L, B, N, R, S, A, md)
    before = e.score(audio)
    e.set_layer_weights(3, w2["Wprev"][3], w2["Wcur"][3], w2["Bh"][3], w2["Wres"][3], w2["Bres"][3], w2["Wskip"][3], w2["Bskip"][3])
    wm = {k: (np.array(v) if isinstance(v, np.ndarray) else v) for k, v in w.items()}
    for k in ("Wprev", "Wcur", "Bh", "Wres", "Bres", "Wskip", "Bskip"):
        wm[k][3] = w2[k][3]
    got = e.score(audio)
    assert not common.bits_equal(before, got)
    assert common.bits_equal(_engine(wm, L, B, N, R, S, A, md).score(audio), got)

    src = _engine(dict(w2, Lh=w["Lh"], selectors=w["selectors"]), L, B, N, R, S, A, md)     # overwrite the blob, then weights_updated
    (ps, n), (pd, nd) = src.weight_blob(), e.weight_blob()
    assert n == nd

    def view(p):
        class _Blob:
            __cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (p, False), "version": 3}
        return torch.as_tensor(_Blob(), device="cuda")
    view(pd).copy_(view(ps)); torch.cuda.synchronize()
    e.weights_updated()
    assert common.bits_equal(src.score(audio), e.score(audio))


@pytest.mark.parametrize("where", ["host", "device"])
def test_errors(where):
    R, S, A, L, B, N, md = 64, 256, 256, 4, 3, 12, 4
    w = refgen.lively_inputs(10, R, S, A, L, B, N)
    e = _engine(w, L, B, N, R, S, A, md)
    good = np.random.default_rng(11).integers(0, A, (B, N)).astype(np.int32)
    bad = good.copy(); bad[1, 7] = A; bad[2, 3] = -1
    put = (lambda a: torch.from_numpy(a).cuda()) if where == "device" else (lambda a: a)
    lib = _lib.lib()
    lp = torch.empty((B, N), device="cuda") if where == "device" else np.empty((B, N), np.float32)
    ptr = lambda a: C.c_void_p(a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data)
    g = put(good)

    def rc(*args):
        return lib.nvwn_score(*args), lib.nvwn_last_error().decode()
    assert rc(None, ptr(g), N, B, ptr(lp), None, None)[0] == EINVAL
    assert rc(e._h, None, N, B, ptr(lp), None, None)[0] == EINVAL
    assert rc(e._h, ptr(g), N, B, None, None, None)[0] == EINVAL
    for bs in (0, B + 1):
        code, msg = rc(e._h, ptr(g), N, bs, ptr(lp), None, None)
        assert code == EINVAL and "batch_size" in msg
    for n in (0, N + 1):
        code, msg = rc(e._h, ptr(g), n, B, ptr(lp), None, None)
        assert code == EINVAL and "num_samples" in msg
    b = put(bad)
    code, msg = rc(e._h, ptr(b), N, B, ptr(lp), None, None)
    assert code == EINVAL and "audio[1][7]" in msg, msg
    with pytest.raises(nw.NvwnError, match=r"audio\[1\]\[7\]"):
        e.score(b)
    ok = e.score(g)                                                     # a valid call still works
    assert common.bits_equal(np.asarray(ok.cpu() if hasattr(ok, "cpu") else ok), e.score(good))
    e32 = nw.NVWavenetInfer(L, md, B, N, R=R, S=S, A=A, dtype=nw.FP32)
    code, msg = rc(e32._h, ptr(g), N, B, ptr(lp), None, None)
    assert code == EUNSUPPORTED and "FP16" in msg
    e512 = nw.NVWavenetInfer(L, md, 1, 4, R=R, S=S, A=512, dtype=nw.FP16)
    code, msg = rc(e512._h, ptr(g), 4, 1, ptr(lp), None, None)
    assert code == EUNSUPPORTED and "A = 256" in msg



def test_device_pointers_streams_and_nvwavenet():
    R, S, A, L, B, N, md = 64, 256, 256, 20, 8, 600, 64
    w = refgen.lively_inputs(12, R, S, A, L, B, N)
    e = _engine(w, L, B, N, R, S, A, md)
    audio = np.random.default_rng(13).integers(0, A, (B, N)).astype(np.int32)
    lp_h, lg_h = e.score(audio, logits=True)
    s = torch.cuda.Stream()
    lp_d, lg_d = e.score(torch.from_numpy(audio).cuda(), logits=True, stream=s)
    s.synchronize()
    assert lp_d.is_cuda and lg_d.is_cuda
    assert common.bits_equal(lp_h, lp_d.cpu().numpy()) and common.bits_equal(lg_h, lg_d.cpu().numpy())

    # NVWaveNet.log_likelihood through its cached fp16 engine, on the same weights as an NVWavenetInfer
    from nv_wavenet_b200.nv_wavenet import NVWaveNet
    g = torch.Generator().manual_seed(14)
    n = lambda *shape, s=0.5: (s * torch.randn(*shape, generator=g)).cuda()
    Lm = 4
    kw = dict(embedding_prev=n(A, R), embedding_curr=n(A, R), conv_out_weight=n(A, S, s=1 / 16), conv_end_weight=n(A, A, s=1 / 8),
              dilate_weights=[n(2 * R, R, 2, s=0.1) for _ in range(Lm)], dilate_biases=[n(2 * R, s=0.1) for _ in range(Lm)],
              max_dilation=8, res_weights=[n(R, R, s=0.1) for _ in range(Lm - 1)], res_biases=[n(R, s=0.05) for _ in range(Lm - 1)],
              skip_weights=[n(S, R, s=0.1) for _ in range(Lm)], skip_biases=[n(S, s=0.05) for _ in range(Lm)], use_embed_tanh=True)
    net = NVWaveNet(**kw)
    Bn, Nn = 3, 50
    cond = n(2 * R, Bn, Lm, Nn)
    aud = torch.randint(0, A, (Bn, Nn), generator=g).to(torch.int32)
    ll = net.log_likelihood(cond, aud)
    assert ll.dtype == torch.float32 and tuple(ll.shape) == (Bn, Nn)
    eng = net._engine(Bn, Nn, True)
    direct = eng.score(aud.numpy())
    assert common.bits_equal(ll.cpu().numpy(), direct)
