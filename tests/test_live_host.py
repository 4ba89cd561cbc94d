"""CPU checks of live vocoding: the frame window of a sample range, the overwrite rule of a push and the ring size against a brute-force
count of the frames upsample_element reads; LiveSession's schedule of pushes and productions against a recording engine; argument
checks that fire before any engine exists; the C++ facade's live members."""
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import nv_wavenet_b200 as nw
from nv_wavenet_b200 import _lib
from nv_wavenet_b200.infer import live_frames, live_push_limit, live_ring_frames
from nv_wavenet_b200.nv_wavenet import LiveSession, NVWaveNet
from tests.test_nv_wavenet_py import _weights

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(12, 5), (4, 2), (800, 200), (7, 7), (9, 4), (5, 1)]          # (upsampling window, stride)


def _read(n, window, stride):
    """the frames upsample_element reads for sample n, in its loop order"""
    out = []
    for m in range(n // stride, -1, -1):
        if n - m * stride >= window:
            break
        out.append(m)
    return out


def test_live_frames_is_the_frames_upsample_element_reads():
    for window, stride in SHAPES:
        for first in range(0, 3 * window + 7):
            for count in (1, 2, stride, window + 3):
                read = {m for n in range(first, first + count) for m in _read(n, window, stride)}
                assert live_frames(first, count, window, stride) == (min(read), max(read) + 1), (window, stride, first, count)


def test_push_limit_keeps_every_frame_a_later_sample_reads():
    for window, stride in SHAPES[:2] + SHAPES[3:]:                      # not C3's: the count takes minutes there
        least = -(-window // stride) + 1
        for ring in (least, least + 3):
            for frames in range(0, 4 * least):
                for produced in range(0, frames * stride + 1):
                    needed = min(m for n in range(produced, produced + 2 * stride) for m in _read(n, window, stride))
                    if frames - ring > needed:                                # a state no accepted push leads to
                        continue
                    # a push of n frames overwrites frames [frames - ring, frames + n - ring)
                    fits = [n for n in range(0, 3 * ring) if frames + n - ring <= needed]
                    assert live_push_limit(frames, produced, ring, window, stride) == max(fits), (window, stride, ring, frames, produced)
                assert live_push_limit(frames, frames * stride, ring, window, stride) >= ring - least + 1 >= 1


def test_ring_frames_holds_a_piece_and_one_more_frame():
    for window, stride in SHAPES:
        for samples in (1, 2, stride, 24, 800):
            span = max(len({m for n in range(first, first + samples) for m in _read(n, window, stride)})      # every first sample mod stride
                       for first in range(window + 2 * stride, window + 3 * stride))
            ring = live_ring_frames(samples, window, stride)
            assert ring == span + 1 and ring >= -(-window // stride) + 1, (window, stride, samples)
    assert live_ring_frames(800, 800, 200) == 9


class _Recorder:
    """an engine that records the live calls a LiveSession makes and checks each against the library's rules"""

    def __init__(self, B, N, window, stride, ring):
        self.B, self.N, self.window, self.stride, self.ring = B, N, window, stride, ring
        self.frames, self.produced, self.generated, self.calls = 0, 0, 0, []

    def cond_producer_push(self, f):
        n = f.shape[2]
        keep = live_frames(self.produced, 1, self.window, self.stride)[0]
        assert self.frames + n - self.ring <= keep, "the library would refuse this push"
        self.frames += n
        self.calls.append(("push", n))

    def cond_producer_run_stream(self, first, m):
        lo, hi = live_frames(first, m, self.window, self.stride)
        assert 1 <= m <= self.N and hi <= self.frames and lo >= self.frames - self.ring
        self.produced = max(self.produced, first + m)
        self.calls.append(("produce", first, m))

    def set_selectors_random_stream(self, seed, first, m):
        self.calls.append(("select", seed, first, m))

    def run_stream(self, first, m, batch):
        assert first == self.generated and batch == self.B and first + m <= self.produced
        self.generated += m
        self.calls.append(("run", first, m))

    def get_yout_stream(self, out, first, m):
        out[:] = torch.arange(first, first + m, dtype=torch.int32)
        return out

    def get_audio_stream(self, first, m, int16=False, saturate=False):
        return np.tile(np.arange(first, first + m), (self.B, 1)).astype(np.int16 if int16 else np.float32)


def test_session_feeds_the_ring_and_generates_each_completed_sample():
    window, stride, W, B = 12, 5, 24, 2
    ring = live_ring_frames(W, window, stride)
    eng = _Recorder(B, W, window, stride, ring)
    live = LiveSession(eng, 3, window, stride, 77, W)
    live.device = "cpu"
    total = 0
    for n in [0, 1, 4, 15, 2, 40, 1]:
        y = live.push(np.zeros((B, 3, n), np.float32))
        assert tuple(y.shape) == (B, n * stride) and torch.equal(y[0], torch.arange(total * stride, (total + n) * stride, dtype=torch.int32))
        total += n
        assert live.frames == eng.frames == total and live.samples == eng.generated == total * stride
    pushes = [c[1] for c in eng.calls if c[0] == "push"]
    assert sum(pushes) == total and max(pushes) == live_push_limit(ring, ring * stride, ring, window, stride) < 15
    runs = [c[1:] for c in eng.calls if c[0] == "run"]
    assert runs == [c[1:] for c in eng.calls if c[0] == "produce"] == [c[2:] for c in eng.calls if c[0] == "select"]
    assert all(m <= W for _, m in runs) and all(c[1] == 77 for c in eng.calls if c[0] == "select")
    y, audio = live.push(np.zeros((B, 3, 2), np.float32), audio="int16")
    assert audio.dtype == np.int16 and np.array_equal(audio[1], y[1].numpy())


def test_push_checks_its_arguments_before_calling_the_engine():
    eng = _Recorder(2, 24, 12, 5, 8)
    live = LiveSession(eng, 3, 12, 5, 0, 24)
    for frames, kw in [(np.zeros((3, 3, 1), np.float32), {}),         # another batch
                       (np.zeros((2, 4, 1), np.float32), {}),         # another channel count
                       (np.zeros((2, 3), np.float32), {}),            # not [batch][C][n]
                       (np.zeros((2, 3, 1), np.float32), {"audio": "int8"})]:
        with pytest.raises(AssertionError):
            live.push(frames, **kw)
    assert eng.calls == [] and live.frames == live.samples == 0


def test_open_live_checks_its_arguments_before_any_engine(monkeypatch):
    lib = _lib.lib()
    R, S, A = lib.get_R(), lib.get_S(), lib.get_A()
    L, Cc, K, stride = 2, 5, 8, 4
    net = NVWaveNet(**_weights(L, R, S, A, np.random.default_rng(5)))
    made = []
    monkeypatch.setattr(net, "_new_engine", lambda *a: made.append(a))
    z = lambda *s: torch.zeros(s)
    good = dict(upsample_weight=z(Cc, Cc, K), upsample_bias=z(Cc), cond_weight=z(L * 2 * R, Cc), cond_bias=z(L * 2 * R), stride=stride,
                batch_size=2, seed=1)
    for kw in [dict(good, upsample_weight=z(Cc, Cc + 1, K)), dict(good, upsample_bias=z(Cc + 1)), dict(good, cond_weight=z(L * 2 * R, Cc - 1)),
               dict(good, cond_bias=z(L * R)), dict(good, stride=K + 1), dict(good, batch_size=0), dict(good, window=0), dict(good, window=None)]:
        with pytest.raises(AssertionError):
            net.open_live(**kw)
    assert made == [] and net.engines_created == 0


def test_null_engine_is_einval():
    lib = _lib.lib()
    assert lib.nvwn_cond_producer_push(None, None, 1, None) == -1
    assert "nvwn_cond_producer_push" in lib.nvwn_last_error().decode()
    assert lib.nvwn_cond_producer_open_live(None, 2, None, None, 4, 2, None, None, 3, None) == -1
    assert "nvwn_cond_producer_open_live" in lib.nvwn_last_error().decode()


def test_cpp_facade_live_members_compile():
    src = r'''
#include "nv_wavenet.hpp"
int main() {
    typedef nvWavenetInfer<float, float, 64, 256, 256> W32;
    typedef nvWavenetInfer<half2, half, 64, 256, 256> W16;
    bool (W16::*open)(int, const float*, const float*, int, int, const float*, const float*, int, cudaStream_t) = &W16::cond_producer_open_live;
    bool (W16::*push)(const float*, int, cudaStream_t) = &W16::cond_producer_push;
    bool (W32::*run)(long long, int, cudaStream_t) = &W32::cond_producer_run_stream;
    (void)open; (void)push; (void)run;
    if (nvwn_device_count() == 0) return 0;
    W32 w(2, 2, 3, 8);
    const int C = 2, K = 4, stride = 2, LR = 2 * 2 * 64;
    std::vector<float> wu(C * C * K, 0.5f), bu(C, 0.1f), wc(LR * C, 0.25f), bc(LR, 0.f), frames(3 * C * 3, 1.f);
    return !w.cond_producer_open_live(C, wu.data(), bu.data(), K, stride, wc.data(), bc.data(), 2) &&
           w.cond_producer_open_live(C, wu.data(), bu.data(), K, stride, wc.data(), bc.data(), 3) && w.cond_producer_push(frames.data(), 3) &&
           w.cond_producer_run_stream(0, 6) && !w.cond_producer_run_stream(0, 7) ? 0 : 1;
}
'''
    with tempfile.TemporaryDirectory() as d:
        f = os.path.join(d, "t.cpp")
        open(f, "w").write(src)
        exe = os.path.join(d, "t")
        cmd = ["g++", "-std=c++14", "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include", f, "-o", exe,
               "-L", os.path.dirname(nw.LIB_PATH), "-lwavenet_infer", "-Wl,-rpath," + os.path.dirname(nw.LIB_PATH)]
        res = subprocess.run(cmd, capture_output=True, text=True)
        assert res.returncode == 0, res.stderr
        assert subprocess.run([exe], capture_output=True).returncode == 0
