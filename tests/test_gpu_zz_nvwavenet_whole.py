"""NVWaveNet's whole-length calls against the engine calls they once made one by one, bit for bit: infer() without a window
against set_conditioning, set_selectors_random (or the libc draw through set_selectors) and run; log_likelihood against
set_conditioning and score; log_likelihood_from_features against set_conditioning_from_features and score.  The calls under test
run the window loop of their windowed forms with one window of the whole length."""
import ctypes as C

import numpy as np
import pytest
import torch

from nv_wavenet_b200 import _lib
from nv_wavenet_b200.nv_wavenet import Impl, column_major
from tests import refgen
from tests.common import bits_equal
from tests.test_gpu_zz_selectors import _net

pytestmark = pytest.mark.gpu

R, S, A, L, MD = 64, 256, 256, 4, 4
# kind -> (fp16, environment, batch, launched kernel)
KINDS = {"fp32": (False, {}, 3, 16), "lat": (True, {}, 3, 18), "tc": (True, {"NVWN_FP16_KERNEL": "tc"}, 64, 17)}
ENV_KEYS = ("NVWN_FP16_KERNEL", "NVWN_LAT_CLUSTER", "NVWN_TC_TILE", "NVWN_TC_NODUP", "NVWN_TC_FUSED", "NVWN_LAT_MAX_B")


def _setup(kind, seed, N, monkeypatch):
    """(fp16, batch, kernel, the network under test, a second network of the same weights for the reference, cond [2R][B][L][N])."""
    fp16, env, B, kernel = KINDS[kind]
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    w = refgen.lively_inputs(seed, R, S, A, L, B, N)
    cond = torch.from_numpy(np.ascontiguousarray(w["Lh"].transpose(3, 2, 1, 0))).cuda()
    return fp16, B, kernel, _net(w, L, R, S, A, MD), _net(w, L, R, S, A, MD), cond


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_infer(kind, monkeypatch):
    N = 300
    fp16, B, kernel, net, ref, cond = _setup(kind, 51, N, monkeypatch)
    libc = C.CDLL(None)
    for seed in (None, 9):
        libc.srand(77)
        got = net.infer(cond, Impl.AUTO, seed=seed, fp16=fp16).cpu().numpy()
        eng = ref._engine(B, N, fp16)
        eng.reset_history()
        eng.set_conditioning(column_major(cond).float(), 0, N)
        if seed is None:
            libc.srand(77)
            sel = np.empty(N * B, np.float32)
            assert _lib.lib().nvwn_libc_selectors(C.c_void_p(sel.ctypes.data), B, N) == 0
            eng.set_selectors(sel)
        else:
            eng.set_selectors_random(seed)
        want = torch.empty((B, N), dtype=torch.int32, device="cuda")
        eng.run(N, B, want)
        torch.cuda.synchronize()
        want = want.cpu().numpy()
        assert len(np.unique(want)) > 8
        assert np.array_equal(got, want), f"seed {seed}: first differences at {np.argwhere(got != want)[:3]}"
    assert net.engines_created == 1 and net._engines[(B, N, fp16)].launch_info()["kernel"] == kernel


@pytest.mark.parametrize("kind", ["lat", "tc"])
def test_log_likelihood(kind, monkeypatch):
    N = 300
    _, B, _, net, ref, cond = _setup(kind, 52, N, monkeypatch)
    audio = torch.from_numpy(np.random.default_rng(52).integers(0, A, (B, N)).astype(np.int32))
    got = net.log_likelihood(cond, audio)
    eng = ref._engine(B, N, True)
    eng.set_conditioning(column_major(cond).float(), 0, N)
    want = eng.score(audio.cuda())
    torch.cuda.synchronize()
    assert torch.isfinite(want).all()
    assert bits_equal(want.cpu().numpy(), got.cpu().numpy())


@pytest.mark.parametrize("kind", ["lat", "tc"])
def test_log_likelihood_from_features(kind, monkeypatch):
    Cc, frames, K, stride = 7, 24, 12, 5
    T = frames * stride
    _, B, _, net, ref, _ = _setup(kind, 53, 1, monkeypatch)
    rng = np.random.default_rng(53)
    features = rng.standard_normal((B, Cc, frames)).astype(np.float32)
    wu = (rng.standard_normal((Cc, Cc, K)) / np.sqrt(Cc * K / stride)).astype(np.float32)
    bu = (0.1 * rng.standard_normal(Cc)).astype(np.float32)
    wc = (0.5 * rng.standard_normal((L * 2 * R, Cc, 1)) / np.sqrt(Cc)).astype(np.float32)
    bc = (0.1 * rng.standard_normal(L * 2 * R)).astype(np.float32)
    audio = rng.integers(0, A, (B, T)).astype(np.int32)
    timing = {}
    got = net.log_likelihood_from_features(features, audio, wu, bu, wc, bc, stride, timing=timing)
    eng = ref._engine(B, T, True)
    eng.set_conditioning_from_features(features, wu, bu, wc.reshape(L * 2 * R, Cc), bc, stride)
    want = eng.score(torch.from_numpy(audio).cuda())
    torch.cuda.synchronize()
    assert torch.isfinite(want).all()
    assert bits_equal(want.cpu().numpy(), got.cpu().numpy())
    assert timing["produce_s"] > 0 and timing["score_s"] > 0
