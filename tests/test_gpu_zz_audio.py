"""Output side on the device (SURVEY.md 8f next-3): nvwn_get_audio decodes the engine's yOut with the reference's
mu-law expansion (pytorch/utils.py:62-70, pytorch/nv_wavenet_inference.py:55-60).  Bit-exact against the oracle:
the device only gathers from a host-computed table."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import mulaw
from tests import refgen

pytestmark = pytest.mark.gpu


def _engine(dtype_name="fp32", B=5, N=48):
    import nv_wavenet_b200 as nw
    L, R, S, A, md = 4, 64, 256, 256, 4
    w = refgen.lively_inputs(11, R, S, A, L, B, N)
    e = nw.NVWavenetInfer(L, md, B, N, R=R, S=S, A=A, dtype=nw.FP16 if dtype_name == "fp16" else nw.FP32)
    e.load(w); e.set_inputs(w["Lh"], w["selectors"])
    y = np.zeros((B, N), np.int32)
    e.run(N, B, y); e.synchronize()
    return e, y


@pytest.mark.parametrize("dtype_name", ["fp32", "fp16"])
def test_audio_matches_oracle(dtype_name):
    e, y = _engine(dtype_name)
    assert y.min() >= 0 and y.max() < 256 and len(np.unique(y)) > 2
    want = mulaw.mu_law_decode(y, 256)
    got = e.get_audio()
    assert got.dtype == np.float32 and got.shape == y.shape
    assert np.array_equal(got, want.astype(np.float32))
    assert np.array_equal(e.get_audio(int16=True), mulaw.to_int16(want))
    assert np.array_equal(e.get_audio(int16=True, saturate=True), mulaw.to_int16(want, saturate=True))
    # a chunk in the middle, as a streaming consumer would ask for it
    assert np.array_equal(e.get_audio(offset=7, size=20), want[:, 7:27].astype(np.float32))
    with pytest.raises(Exception):
        e.get_audio(offset=40, size=20)                                    # out of range
    with pytest.raises(ValueError):
        e.get_audio(size=20, out=np.empty((y.shape[0], 10), np.float32))   # a buffer too small for B x size values


def test_audio_into_device_tensor_on_a_stream():
    import torch
    e, y = _engine()
    st = torch.cuda.Stream()
    out = torch.empty((y.shape[0], 16), dtype=torch.int16, device="cuda")
    e.get_audio(offset=32, size=16, int16=True, out=out, stream=st)
    st.synchronize()
    assert np.array_equal(out.cpu().numpy(), mulaw.to_int16(mulaw.mu_law_decode(y[:, 32:48], 256)))


def test_caller_arrays_are_checked_under_python_O():
    """The checks on a caller's buffer (get_audio's out) and arrays (the features of the whole-batch producer) are raised
    ValueErrors, so `python -O` keeps them: without them the library writes or reads past the caller's memory."""
    code = """if True:
        import numpy as np
        import nv_wavenet_b200 as nw
        e = nw.NVWavenetInfer(2, 2, 2, 16, R=64, S=256, A=256, dtype=nw.FP32)
        net = (np.zeros((3, 3, 8), np.float32), np.zeros(3, np.float32), np.zeros((256, 3), np.float32), np.zeros(256, np.float32), 4)
        calls = {"get_audio": lambda: e.get_audio(0, 16, out=np.empty((2, 8), np.float32)),
                 "set_conditioning_from_features": lambda: e.set_conditioning_from_features(np.zeros((3, 3, 4), np.float32), *net)}
        for name, call in calls.items():
            try:
                call()
            except ValueError:
                continue
            raise SystemExit(name + " raised no ValueError under -O")
        print("ok")
    """
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    flags = ["-O"] + (["-s"] if sys.flags.no_user_site else [])
    out = subprocess.run([sys.executable, *flags, "-c", code], capture_output=True, text=True, timeout=300, cwd=root)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr[-2000:]
