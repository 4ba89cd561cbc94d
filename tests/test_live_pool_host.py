"""CPU checks of live serving: the step planner (plan_live_step) over scripted frame arrivals -- stalls, bursts, early finishes and more
streams than slots -- and a LivePool driven through a recording engine that applies the library's per-slot live and slot-state rules;
argument checks before any engine exists; NULL engines; the C++ facade's new members."""
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

import nv_wavenet_b200 as nw
from nv_wavenet_b200 import _lib
from nv_wavenet_b200.infer import live_frames, live_ring_frames
from nv_wavenet_b200.nv_wavenet import LivePool, NVWaveNet, live_ready, plan_live_step
from tests.test_nv_wavenet_py import _weights

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _script(rng, n_streams, steps, stride):
    """per stream (open step, [frames arriving at each step], finish step): some stall for several steps, some arrive in bursts, some
    finish early"""
    out = []
    for i in range(n_streams):
        opened = int(rng.integers(0, steps // 3))
        total = int(rng.integers(1, 12))
        arrivals = np.zeros(steps, np.int64)
        t = opened
        left = total
        while left > 0 and t < steps:
            if rng.random() < 0.25:
                t += int(rng.integers(2, 5))                           # a stall
                continue
            n = min(left, int(rng.integers(1, 5)) if rng.random() < 0.8 else left)     # a burst: everything at once
            arrivals[t] += n
            left -= n
            t += 1
        out.append((opened, arrivals, min(t, steps - 1) if left == 0 else None))
    return out


def test_planner_over_scripted_arrivals():
    """No slot is used twice, only ready streams run, ready waiting streams are served FIFO, and every stream completes once its
    frames are in, over random scripts of more streams than slots."""
    window, stride = 6, 2
    for seed in range(40):
        rng = np.random.default_rng(seed)
        slots = int(rng.integers(1, 5))
        script = _script(rng, int(rng.integers(slots, 3 * slots + 3)), 60, stride)
        pos, frames, fin, slot = {}, {}, {}, {}
        waiting, done = [], set()
        for step in range(400):
            for i, (opened, arrivals, finish) in enumerate(script):
                if opened == step:
                    pos[i], frames[i], fin[i], slot[i] = 0, 0, False, None
                    waiting.append(i)
                if i in frames and step < len(arrivals):
                    frames[i] += int(arrivals[step])
                if finish == step:
                    fin[i] = True
            resident = {i: (slot[i], pos[i], frames[i], fin[i]) for i in slot if slot[i] is not None and i not in done}
            park, place = plan_live_step(resident, [(i, pos[i], frames[i], fin[i]) for i in waiting], slots, window, stride)
            for i in park:
                assert not live_ready(pos[i], frames[i], fin[i], window, stride)
                slot[i] = None
                waiting.append(i)
            ready_waiting = [i for i in waiting if i not in park and live_ready(pos[i], frames[i], fin[i], window, stride)]
            assert [i for i, _ in place] == ready_waiting[:len(place)], "ready streams take slots in the order they began to wait"
            for i, b in place:
                slot[i] = b
                waiting.remove(i)
            running = [i for i in slot if slot[i] is not None and i not in done]
            used = [slot[i] for i in running]
            assert len(used) == len(set(used)) and all(0 <= b < slots for b in used), "a slot is used twice"
            if len(running) < slots:
                assert not any(live_ready(pos[i], frames[i], fin[i], window, stride) for i in waiting), "a ready stream waits by a free slot"
            for i in running:
                assert live_ready(pos[i], frames[i], fin[i], window, stride), "a stream runs that is not ready"
                pos[i] += min(window, frames[i] * stride - pos[i])
                if fin[i] and pos[i] == frames[i] * stride:
                    done.add(i)
                    slot[i] = None
            for i in list(waiting):                                     # finish() of a stream with nothing left
                if fin[i] and pos[i] == frames[i] * stride:
                    waiting.remove(i)
                    done.add(i)
        finished = {i for i, (_, _, f) in enumerate(script) if f is not None}
        assert finished <= done, (seed, finished - done)
        for i in finished:
            assert pos[i] == frames[i] * stride


def test_planner_parks_and_frees():
    # slot 0's stream stalls; slot 1's is ready; two wait, the first not ready
    park, place = plan_live_step({0: (0, 6, 3, False), 1: (1, 0, 5, False)}, [(2, 0, 1, False), (3, 0, 4, False), (4, 0, 0, True)], 2, 6, 2)
    assert park == [0] and place == [(3, 0)]
    # a finished stream with samples left is ready however few
    assert plan_live_step({}, [(7, 10, 6, True)], 1, 6, 2) == ([], [(7, 0)])
    assert plan_live_step({}, [(7, 12, 6, True)], 1, 6, 2) == ([], [])


class _PoolEngine:
    """an engine that records what a LivePool does and checks each call against the library's rules: per-slot live rings (attach,
    push, produce), restarts and slot states (save at the engine's next sample, load with origin t0 - position)"""

    def __init__(self, B, N, K, stride):
        self.B, self.N, self.K, self.stride = B, N, K, stride
        self.t, self.ring, self.calls = 0, None, []
        self.slot = [None] * B                   # per slot: dict(start, first, T, done, origin, seed) or None
        self.saved = {}

    def cond_producer_open_live_slots(self, ring):
        self.ring = ring

    def restart_slots(self, slots, seeds):
        for b, s in zip(slots, seeds):
            self.slot[b] = dict(start=None, first=0, T=0, done=0, origin=self.t, seed=s)
        self.calls.append(("restart", list(slots)))

    def save_slots(self, slots):
        out = torch.zeros((len(slots), 2), dtype=torch.int64)
        for j, b in enumerate(slots):
            out[j, 0] = self.t - self.slot[b]["origin"]            # the position the state records
            out[j, 1] = self.slot[b]["seed"]
            self.slot[b] = None
        self.calls.append(("save", list(slots), out[:, 0].tolist()))
        return out

    def load_slots(self, slots, states):
        for b, st in zip(slots, states):
            self.slot[b] = dict(start=None, first=0, T=0, done=0, origin=self.t - int(st[0]), seed=int(st[1]))
        self.calls.append(("load", list(slots), [int(st[0]) for st in states]))

    def cond_producer_attach_live(self, slots, starts, first_frames, features):
        for b, start, first, f in zip(slots, starts, first_frames, features):
            s = self.slot[b]
            assert start == s["origin"], "the utterance's sample 0 must sit at its selector origin"
            assert 0 <= f.shape[1] <= self.ring
            s.update(start=start, first=first, T=first + f.shape[1], done=0)
        self.calls.append(("attach", list(slots), list(starts), list(first_frames)))

    def cond_producer_push_slots(self, slots, features):
        for b, f in zip(slots, features):
            s = self.slot[b]
            keep = max(s["first"], live_frames(s["done"], 1, self.K, self.stride)[0])
            assert s["T"] + f.shape[1] - self.ring <= keep, "the library would refuse this push"
            s["T"] += f.shape[1]
        self.calls.append(("push", list(slots), [f.shape[1] for f in features]))

    def cond_producer_run_slots(self, slots, first, n):
        assert first == self.t and n == self.N
        for b in slots:
            s = self.slot[b]
            n0 = first - s["start"]
            assert n0 >= 0
            if n0 < s["T"] * self.stride:
                assert live_frames(n0, 1, self.K, self.stride)[0] >= max(s["first"], s["T"] - self.ring), "a frame has left the ring"
            s["done"] = max(s["done"], n0 + n)
        self.run_slots = list(slots)

    def set_selectors_random_slots(self, first, n):
        pass

    def run_stream(self, first, n, batch):
        assert first == self.t and batch == self.B
        self.t += n
        self.calls.append(("run", first, sorted(self.run_slots)))

    def get_yout(self, stage, pos, n):
        # row b: the utterance-local sample index of each sample, so the pool's outputs read back as 0, 1, 2, ...
        for b in range(self.B):
            if self.slot[b] is not None and self.slot[b]["start"] is not None:
                stage[b, pos:pos + n] = torch.arange(self.t - n, self.t, dtype=torch.int32) - self.slot[b]["start"]
            else:
                stage[b, pos:pos + n] = -1


def test_pool_schedule_against_a_recording_engine():
    """7 streams on 3 slots with stalls and a late opener: each stream's outputs are its samples 0 .. n - 1 in order, with every
    sample its frames complete; parked streams resume with start = t - position, from the first frame sample `position` reads."""
    K, stride, W, B = 12, 5, 10, 3
    eng = _PoolEngine(B, W, K, stride)
    pool = LivePool(eng, 2, K, stride)
    pool.device = "cpu"
    assert eng.ring == live_ring_frames(W, K, stride) == pool.ring_frames
    rng = np.random.default_rng(3)
    totals = [9, 14, 4, 11, 7, 20, 6]
    ids, got, given = [], {}, {}
    for i in range(7):
        if i < 6:
            ids.append(pool.open(100 + i))
    stalls = {1: range(3, 9), 3: range(2, 12), 5: range(5, 7)}
    for step in range(200):
        if step == 4:
            ids.append(pool.open(106))                                  # opens late
        for j, i in enumerate(ids):
            if j in stalls and step in stalls[j]:
                continue
            n = min(int(rng.integers(0, 3)), totals[j] - given.get(i, 0))
            if n:
                pool.push(i, np.zeros((2, n), np.float32))
                given[i] = given.get(i, 0) + n
            elif given.get(i, 0) == totals[j] and i in pool._streams and not pool._streams[i].finished:
                pool.finish(i)
        for i, y in pool.step().items():
            got.setdefault(i, []).append(y)
        if not pool._streams:
            break
    assert not pool._streams and pool.parks > 0 and pool.resumes > 0 and pool.launches == len([c for c in eng.calls if c[0] == "run"])
    for j, i in enumerate(ids):
        y = torch.cat(got[i])
        assert torch.equal(y, torch.arange(totals[j] * stride, dtype=torch.int32)), (j, y)
    for c in eng.calls:
        if c[0] == "run":
            assert len(c[2]) == len(set(c[2])) <= B
    # every load is followed by an attach of those slots at start t - position, from the first frame sample `position` reads
    for k, c in enumerate(eng.calls):
        if c[0] == "load":
            att = next(a for a in eng.calls[k + 1:] if a[0] == "attach")
            for b, p in zip(c[1], c[2]):
                j = att[1].index(b)
                run = next(r for r in eng.calls[k:] if r[0] == "run")
                assert att[2][j] == run[1] - p and att[3][j] == live_frames(p, 1, K, stride)[0]


def test_pool_checks_its_arguments():
    eng = _PoolEngine(2, 10, 12, 5)
    pool = LivePool(eng, 3, 12, 5)
    i = pool.open(1)
    for call in (lambda: pool.push(i, np.zeros((4, 1), np.float32)), lambda: pool.push(i + 1, np.zeros((3, 1), np.float32)),
                 lambda: pool.step(audio="int8")):
        with pytest.raises(AssertionError):
            call()
    pool.finish(i)                                                      # nothing pushed: the stream leaves at once
    assert pool.step() == {} and pool.launches == 0 and eng.calls == []
    with pytest.raises(AssertionError):
        pool.push(i, np.zeros((3, 1), np.float32))


def test_open_live_pool_checks_its_arguments_before_any_engine(monkeypatch):
    lib = _lib.lib()
    R, S, A = lib.get_R(), lib.get_S(), lib.get_A()
    L, Cc, K, stride = 2, 5, 8, 4
    net = NVWaveNet(**_weights(L, R, S, A, np.random.default_rng(5)))
    made = []
    monkeypatch.setattr(net, "_new_engine", lambda *a: made.append(a))
    z = lambda *s: torch.zeros(s)
    good = dict(upsample_weight=z(Cc, Cc, K), upsample_bias=z(Cc), cond_weight=z(L * 2 * R, Cc), cond_bias=z(L * 2 * R), stride=stride,
                slots=2, window=8)
    for kw in [dict(good, upsample_weight=z(Cc, Cc + 1, K)), dict(good, cond_bias=z(L * R)), dict(good, stride=K + 1), dict(good, slots=0),
               dict(good, window=0), dict(good, window=None)]:
        with pytest.raises(AssertionError):
            net.open_live_pool(**kw)
    assert made == []


def test_null_engine_is_einval():
    lib = _lib.lib()
    for name, args in [("nvwn_slot_state_bytes", (None, None)), ("nvwn_save_slots", (None, None, 1, None, None)),
                       ("nvwn_load_slots", (None, None, 1, None, None)), ("nvwn_cond_producer_open_live_slots", (None, 4, None)),
                       ("nvwn_cond_producer_attach_live", (None, None, 1, None, None, None, None, None)),
                       ("nvwn_cond_producer_push_slots", (None, None, 1, None, None, None))]:
        assert getattr(lib, name)(*args) == -1
        assert name in lib.nvwn_last_error().decode()


def test_cpp_facade_slot_state_members_compile():
    src = r'''
#include "nv_wavenet.hpp"
int main() {
    typedef nvWavenetInfer<half2, half, 64, 256, 256> W16;
    static_assert(sizeof(nvwn_slot_state_header) == 64, "header");
    unsigned long long (W16::*bytes)() = &W16::slot_state_bytes;
    bool (W16::*save)(const int*, int, void*, cudaStream_t) = &W16::save_slots;
    bool (W16::*load)(const int*, int, const void*, cudaStream_t) = &W16::load_slots;
    bool (W16::*open)(int, cudaStream_t) = &W16::cond_producer_open_live_slots;
    bool (W16::*attach)(const int*, int, const long long*, const int*, const float* const*, const int*, cudaStream_t) = &W16::cond_producer_attach_live;
    bool (W16::*push)(const int*, int, const float* const*, const int*, cudaStream_t) = &W16::cond_producer_push_slots;
    (void)bytes; (void)save; (void)load; (void)open; (void)attach; (void)push;
    return 0;
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
