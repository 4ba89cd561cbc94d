"""Numerical contract of a fused tensor-core layer schedule, explored on the CPU.

A fused schedule (one MMA <-> epilogue round trip per layer) does not evaluate the layer the way the reference writes it
(nv_wavenet_reference.cpp:59-86): it folds Wf_l = Wcur_l . Wres_{l-1} (one fp16 matrix) and
Bh'_l = Bh_l + Wcur_l . Bres_{l-1}, accumulates a_l = (Lh + Bh') + Wprev.x_l[t-d] + Wcur.x_{l-1} + Wf.h_{l-1}, and
evaluates tanh / sigmoid on fp16 values.  This test restates that arithmetic in numpy (fp16 roundings where the kernel
has them, fp32 accumulation), teacher-forced on the fp32 oracle's trajectory, and checks over several seeds and shapes
that its logits stay within the north-star tolerance (1e-2 relative, same criterion as tests/test_gpu_parity.py) of the
fp32 oracle -- i.e. that the algebraic fold costs no accuracy class.  The unfused fp16 contract is run alongside as
a yardstick."""
import numpy as np
import pytest

from oracle import pyoracle as po
from tests import refgen

f16 = lambda a: np.asarray(a, np.float32).astype(np.float16).astype(np.float32)


def dilations(L, md):
    out, d = [], 1
    for _ in range(L):
        out.append(d)
        d = d * 2 if d * 2 <= md else 1
    return out


def logits(w, L, B, N, R, S, A, md, forced, mode):
    """Za [B][A] of the last sample; mode in {"fp32", "fp16", "fused"}; weights are column-major flats (tests/refgen.py)."""
    q = (lambda a: np.asarray(a, np.float32)) if mode == "fp32" else f16
    mat = lambda flat, M, K: q(flat).reshape(K, M).T                     # column-major flat -> [M][K]
    Wprev = [mat(w["Wprev"][l], 2 * R, R) for l in range(L)]; Wcur = [mat(w["Wcur"][l], 2 * R, R) for l in range(L)]
    Wres = [mat(w["Wres"][l], R, R) for l in range(L)]; Wskip = [mat(w["Wskip"][l], S, R) for l in range(L)]
    Bh, Bres, Bskip = q(w["Bh"]), q(w["Bres"]), q(w["Bskip"])
    Wzs, Wza, Bzs, Bza = mat(w["Wzs"], A, S), mat(w["Wza"], A, A), q(w["Bzs"]), q(w["Bza"])
    embP, embC, Lh = q(w["embPrev"]), q(w["embCur"]), q(w["Lh"])
    dil = dilations(L, md)
    if mode == "fused":
        Wf = [None] + [f16(Wcur[l] @ Wres[l - 1]) for l in range(1, L)]
        Bhf = [Bh[0]] + [Bh[l] + Wcur[l] @ Bres[l - 1] for l in range(1, L)]
    hist = np.zeros((N, L, B, R), np.float32)                            # x_l[t], as the GEMM input the kernel stores (fp16 unless fp32 mode)
    yp = np.full(B, 128); yc = np.full(B, 128)
    sig = lambda v: 1.0 / (1.0 + np.exp(-v))
    za = None
    for t in range(N):
        x = np.tanh(embP[yp] + embC[yc]).astype(np.float32)             # [B][R]
        skip = np.zeros((B, S), np.float32)
        h_prev = x_prev_in = None
        for l in range(L):
            xin = q(x)
            hist[t, l] = xin
            a = Lh[t, l] + (Bhf[l] if mode == "fused" else Bh[l])
            if t >= dil[l]:
                a = a + hist[t - dil[l], l] @ Wprev[l].T
            if mode == "fused" and l > 0:
                a = a + x_prev_in @ Wcur[l].T + h_prev @ Wf[l].T
            else:
                a = a + xin @ Wcur[l].T
            a = a.astype(np.float32)
            if mode == "fused":
                th = f16(np.tanh(f16(a[:, :R]))); tg = f16(np.tanh(f16(0.5 * a[:, R:])))
                h = f16(th * f16(0.5 * tg + 0.5))
            else:
                h = q(np.tanh(a[:, :R]) * sig(a[:, R:]))
            skip = skip + h @ Wskip[l].T + Bskip[l]
            x_prev_in, h_prev = xin, h
            x = (x + (h @ Wres[l].T + Bres[l])).astype(np.float32)
        zs = np.maximum(q(np.maximum(skip, 0)) @ Wzs.T + Bzs, 0)
        za = q(zs) @ Wza.T + Bza
        yp, yc = yc, forced[:, t]
    return za.astype(np.float32)


def check(za_ref, za, rel=1e-2):
    scale = np.abs(za_ref).max(axis=-1, keepdims=True)
    err = np.abs(za - za_ref)
    assert np.all(err <= rel * np.maximum(np.abs(za_ref), 0.25 * scale)), (err / scale).max()
    return float((err / scale).max()), float((err / scale).mean())


@pytest.mark.parametrize("seed,shape", [(s, sh) for s in range(4) for sh in [(64, 256, 256, 20, 2, 24, 8), (64, 128, 256, 12, 3, 20, 512)]])
def test_fused_contract_stays_within_the_north_star_tolerance(seed, shape):
    R, S, A, L, B, N, md = shape
    w = refgen.lively_inputs(300 + seed, R, S, A, L, B, N)
    o = po.Oracle(L, B, N, R, S, A, md, math=po.MATH_PORTABLE, prec=po.PREC_FP32, tanh_embed=True)
    o.load(w); o.set_inputs(w["Lh"], w["selectors"])
    forced = o.run(N, B)
    o2 = po.Oracle(L, B, N, R, S, A, md, math=po.MATH_PORTABLE, prec=po.PREC_FP32, tanh_embed=True)
    o2.load(w); o2.set_inputs(w["Lh"], w["selectors"]); o2.set_forced(forced); o2.run(N, B)
    za_ref = o2.get_za()
    # the numpy restatement in fp32 must reproduce the C oracle (validates the restatement itself)
    za32 = logits(w, L, B, N, R, S, A, md, forced, "fp32")
    assert np.abs(za32 - za_ref).max() <= 2e-4 * np.abs(za_ref).max()
    m16, a16 = check(za_ref, logits(w, L, B, N, R, S, A, md, forced, "fp16"))
    mfu, afu = check(za_ref, logits(w, L, B, N, R, S, A, md, forced, "fused"))
    # the fold may cost a little but not an accuracy class: within 3x of the unfused fp16 contract's own error
    assert mfu <= max(3 * m16, 2e-3) and afu <= max(3 * a16, 5e-4), (m16, a16, mfu, afu)
