"""CPU check that the serving calls of nv_wavenet.py -- NVWaveNet's infer, infer_many, infer_many_from_features and log_likelihood
family, ModelSet.infer_many, LiveSession and LivePool -- make the engine calls they made when tests/golden/serving_calls.json was
written: every NVWavenetInfer method with its arguments (tensors and arrays by dtype, shape and a hash of their bytes), the stream
each is enqueued on, the cross-stream event records and waits between them, the synchronises, where each timing event is
recorded and which pairs of them each `timing` key sums, and a hash of each public call's result.  The engine is a recording one that writes deterministic values into everything the layer reads back;
torch.cuda's streams, events and synchronise are replaced by recording stand-ins and CUDA tensors are made on the CPU.
tests/golden/make_serving_calls.py rewrites the golden file."""
import contextlib
import ctypes
import hashlib
import inspect
import json
import os

import numpy as np
import torch

from nv_wavenet_b200 import _lib
from nv_wavenet_b200.infer import NVWavenetInfer
from nv_wavenet_b200.nv_wavenet import ModelSet, NVWaveNet

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "serving_calls.json")


def _hash(b):
    return hashlib.sha256(b).hexdigest()[:16]


class _Log:
    """what one case did: its calls in order, the labels of its engines and streams, and the timing events it created"""

    def __init__(self):
        self.calls, self.engines, self.streams, self.events, self.timing_events = [], 0, 0, 0, 0

    def enc(self, v):
        if isinstance(v, torch.Tensor):
            return ["tensor", str(v.dtype), list(v.shape), _hash(v.detach().contiguous().cpu().numpy().tobytes())]
        if isinstance(v, np.ndarray):
            return ["array", str(v.dtype), list(v.shape), _hash(np.ascontiguousarray(v).tobytes())]
        if isinstance(v, (_Stream, _Event, _Engine)):
            return v.label
        if isinstance(v, (list, tuple)):
            return [self.enc(x) for x in v]
        if isinstance(v, dict):
            return {str(k): self.enc(x) for k, x in v.items()}
        if isinstance(v, (bool, str)) or v is None:
            return v
        if isinstance(v, (int, np.integer)):
            return int(v)
        if isinstance(v, (float, np.floating)):
            return float(v)
        raise TypeError(f"cannot record a {type(v)}")


LOG = None


class _Stream:
    def __init__(self, label):
        self.label = label

    def wait_event(self, ev):
        LOG.calls.append(["wait_event", self.label, ev.label])

    def wait_stream(self, other):
        LOG.calls.append(["wait_stream", self.label, other.label])


def _current():
    return _CURRENT


def _default():
    return _DEFAULT


_CURRENT, _DEFAULT = _Stream("stream:current"), _Stream("stream:default")


def _new_stream(*a, **k):
    LOG.streams += 1
    return _Stream(f"stream:side-{LOG.streams}")


class _Event:
    """events are labelled in creation order, timing ones apart, and their records logged; the elapsed time between two timing
    events is logged and is the difference of their numbers in ms, so a sum of spans tells which spans it summed"""

    def __init__(self, enable_timing=False, **k):
        self.timing = enable_timing
        if enable_timing:
            LOG.timing_events += 1
            self.n, self.label = LOG.timing_events, f"timing-{LOG.timing_events}"
        else:
            LOG.events += 1
            self.label = f"event-{LOG.events}"

    def record(self, stream=None):
        LOG.calls.append(["record", self.label, (stream or _CURRENT).label])

    def elapsed_time(self, other):
        assert self.timing and other.timing
        LOG.calls.append(["elapsed_time", self.label, other.label])
        return float(other.n - self.n)


def _synchronize(*a):
    LOG.calls.append(["synchronize"])


_OUT = {"get_yout": "y_out", "get_yout_stream": "out"}          # arguments the engine writes: recorded by dtype and shape only


class _Engine:
    """records every call with its arguments bound to NVWavenetInfer's signature; writes deterministic values into what it returns"""

    def __init__(self, batch_size, sample_count, fp16):
        LOG.engines += 1
        self.label = f"engine-{LOG.engines}"
        self.B, self.N, self.A = batch_size, sample_count, 256
        self.dtype = _lib.FP16 if fp16 else _lib.FP32
        self.model_group = 2
        self.k = 0
        LOG.calls.append(["new_engine", self.label, batch_size, sample_count, bool(fp16)])

    def _values(self, shape, mod):
        self.k += 1
        return (np.arange(int(np.prod(shape)), dtype=np.int64).reshape(shape) * 7 + self.k * 31) % mod

    def __getattr__(self, name):
        real = getattr(NVWavenetInfer, name, None)
        if real is None or name.startswith("_"):
            raise AttributeError(name)
        sig = inspect.signature(real)

        def call(*args, **kwargs):
            bound = sig.bind(self, *args, **kwargs)
            bound.apply_defaults()
            bound.arguments.pop("self")
            rec = {}
            for k, v in bound.arguments.items():
                if _OUT.get(name) == k:
                    rec[k] = ["out", str(v.dtype), list(v.shape)]
                else:
                    rec[k] = LOG.enc(v)
            LOG.calls.append([name, self.label, rec])
            return getattr(self, "_ret_" + name, lambda **kw: None)(**bound.arguments)
        return call

    def _ret_get_yout(self, y_out, offset, size, **k):
        y_out[:, offset:offset + size] = torch.from_numpy(self._values((y_out.shape[0], size), 256)).to(torch.int32)

    def _ret_get_yout_stream(self, out, count, **k):
        out[:, :count] = torch.from_numpy(self._values((out.shape[0], count), 256)).to(torch.int32)
        return out

    def _ret_get_audio(self, size, int16, **k):
        v = self._values((self.B, size), 65536)
        return (v - 32768).astype(np.int16) if int16 else (v / 65536).astype(np.float32)

    def _ret_get_audio_stream(self, count, int16, **k):
        return self._ret_get_audio(count, int16)

    def _ret_score_stream(self, audio, num_samples, batch_size, **k):
        shape = (audio.shape[0] if batch_size is None else batch_size, audio.shape[1] if num_samples is None else num_samples)
        return -torch.from_numpy(self._values(shape, 1000)).to(torch.float32) / 100

    def _ret_score_stream_packed(self, audio, num_samples, batch_size, **k):
        return self._ret_score_stream(audio, num_samples, batch_size)

    def _ret_save_slots(self, slots, **k):
        return torch.from_numpy(self._values((len(slots), 16), 256)).to(torch.uint8)

    def _ret_score_save_states(self, rows, **k):
        return self._ret_save_slots(rows)


def _cpu(device):
    if isinstance(device, torch.device):
        return torch.device("cpu") if device.type == "cuda" else device
    return "cpu" if isinstance(device, str) and device.startswith("cuda") else device


def _on_cpu_factory(fn):
    def f(*a, **k):
        if "device" in k:
            k["device"] = _cpu(k["device"])
        return fn(*a, **k)
    return f


@contextlib.contextmanager
def recording():
    """the stand-ins of torch.cuda and of NVWaveNet._new_engine, undone on exit"""
    saved = []

    def patch(obj, name, value):
        saved.append((obj, name, obj.__dict__[name] if name in obj.__dict__ else getattr(obj, name)))
        setattr(obj, name, value)

    real_to = torch.Tensor.to

    def to(self, *a, **k):
        a = tuple(_cpu(x) for x in a)
        if "device" in k:
            k["device"] = _cpu(k["device"])
        return real_to(self, *a, **k)

    try:
        for name in ("empty", "zeros", "full", "tensor", "as_tensor", "arange"):
            patch(torch, name, _on_cpu_factory(getattr(torch, name)))
        patch(torch.Tensor, "to", to)
        patch(torch.cuda, "Event", _Event)
        patch(torch.cuda, "Stream", _new_stream)
        patch(torch.cuda, "current_stream", _current)
        patch(torch.cuda, "default_stream", _default)
        patch(torch.cuda, "synchronize", _synchronize)
        patch(NVWaveNet, "_new_engine", lambda self, b, n, fp16: _Engine(b, n, fp16))
        yield
    finally:
        for obj, name, value in reversed(saved):
            setattr(obj, name, value)


# ---- the cases ----

def _lib_dims():
    lib = _lib.lib()
    return lib.get_R(), lib.get_S(), lib.get_A()


def _net(seed, L=2):
    R, S, A = _lib_dims()
    rng = np.random.default_rng(seed)
    t = lambda *s: torch.from_numpy(rng.standard_normal(s).astype(np.float32))
    return NVWaveNet(embedding_prev=t(A, R), embedding_curr=t(A, R), conv_out_weight=t(A, S, 1), conv_end_weight=t(A, A, 1),
                     dilate_weights=[t(2 * R, R, 2) for _ in range(L)], dilate_biases=[t(2 * R) for _ in range(L)], max_dilation=4,
                     res_weights=[t(R, R, 1) for _ in range(L - 1)], res_biases=[t(R) for _ in range(L - 1)],
                     skip_weights=[t(S, R, 1) for _ in range(L)], skip_biases=[t(S) for _ in range(L)], use_embed_tanh=False)


L, CC, K, STRIDE = 2, 3, 8, 4


def _f32(rng, *s):
    return rng.standard_normal(s).astype(np.float32)


def _codes(rng, *s):
    return torch.from_numpy(rng.integers(0, 256, s).astype(np.int32))


def _network(rng):
    R = _lib_dims()[0]
    return dict(upsample_weight=torch.from_numpy(_f32(rng, CC, CC, K)), upsample_bias=torch.from_numpy(_f32(rng, CC)),
                cond_weight=torch.from_numpy(_f32(rng, L * 2 * R, CC, 1)), cond_bias=torch.from_numpy(_f32(rng, L * 2 * R)), stride=STRIDE)


def _srand(seed):
    ctypes.CDLL(None).srand(seed)


def _infer(window, seed, fp16, P):
    def run():
        R = _lib_dims()[0]
        rng = np.random.default_rng(1)
        net = _net(0)
        cond = torch.from_numpy(_f32(rng, 2 * R, 2, L, 21))
        _srand(11)
        prompt = None if P is None else _codes(rng, 2, P)
        return net.infer(cond, 0, seed=seed, fp16=fp16, window=window, prompt=prompt), None
    return run


def _infer_many(prompted, timed):
    def run():
        R = _lib_dims()[0]
        rng = np.random.default_rng(2)
        lengths = [20, 13, 30, 9, 17, 25, 12]
        conds = [torch.from_numpy(_f32(rng, 2 * R, L, n)) for n in lengths]
        # two prompts of 5 samples, one that ends on the window boundary 8, one of 11
        prompts = [None, _codes(rng, 5), _codes(rng, 5), _codes(rng, 8), None, _codes(rng, 11), None] if prompted else None
        timing = {} if timed else None
        out = _net(0).infer_many(conds, [100 + u for u in range(len(lengths))], slots=3, window=8, fp16=prompted, timing=timing,
                                 prompts=prompts)
        return out, timing
    return run


def _infer_many_from_features(as_torch):
    def run():
        rng = np.random.default_rng(3)
        frames = [_f32(rng, CC, T) for T in (5, 3, 7, 2, 4)]
        if as_torch:
            frames = [torch.from_numpy(f) for f in frames]
        timing = {}
        out = _net(0).infer_many_from_features(frames, [7, 8, 9, 10, 11], **_network(rng), slots=2, window=8, timing=timing)
        return out, timing
    return run


def _log_likelihood(window):
    def run():
        R = _lib_dims()[0]
        rng = np.random.default_rng(4)
        return _net(0).log_likelihood(torch.from_numpy(_f32(rng, 2 * R, 2, L, 19)), _codes(rng, 2, 19), window=window), None
    return run


def _log_likelihood_from_features(window, timed):
    def run():
        rng = np.random.default_rng(5)
        timing = {} if timed else None
        out = _net(0).log_likelihood_from_features(_f32(rng, 2, CC, 5), _codes(rng, 2, 5 * STRIDE), **_network(rng), window=window,
                                                   timing=timing)
        return out, timing
    return run


def _log_likelihood_many(timed):
    def run():
        R = _lib_dims()[0]
        rng = np.random.default_rng(6)
        lengths = [11, 4, 19, 7, 9]
        timing = {} if timed else None
        out = _net(0).log_likelihood_many([torch.from_numpy(_f32(rng, 2 * R, L, n)) for n in lengths], [_codes(rng, n) for n in lengths],
                                          slots=2, window=8, timing=timing)
        return out, timing
    return run


def _log_likelihood_many_from_features(timed):
    def run():
        rng = np.random.default_rng(7)
        T = [3, 1, 4, 2, 2]
        timing = {} if timed else None
        out = _net(0).log_likelihood_many_from_features([_f32(rng, CC, t) for t in T], [_codes(rng, t * STRIDE) for t in T],
                                                        **_network(rng), slots=2, window=8, timing=timing)
        return out, timing
    return run


def _model_set(timed):
    def run():
        R = _lib_dims()[0]
        rng = np.random.default_rng(8)
        lengths = [20, 13, 30, 9, 17, 25, 12]
        ms = ModelSet([_net(0), _net(1), _net(2)])
        timing = {} if timed else None
        out = ms.infer_many([0, 1, 2, 1, 0, 2, 2], [torch.from_numpy(_f32(rng, 2 * R, L, n)) for n in lengths],
                            [50 + u for u in range(len(lengths))], slots=4, window=8, timing=timing)
        ms.close()
        return out, timing
    return run


def _live(P, audio):
    def run():
        rng = np.random.default_rng(9)
        prompt = None if P is None else _codes(rng, 2, P)
        s = _net(0).open_live(**_network(rng), batch_size=2, seed=5, window=8, fp16=P is not None, prompt=prompt)
        outs = []
        for n in (1, 0, 3, 2, 7, 1, 4):
            outs.append(s.push(_f32(rng, 2, CC, n), audio=audio))
        s.close()
        return outs, None
    return run


def _pool_stalls(audio, timed):
    """7 streams on 3 slots with stalls and a late opener (test_live_pool_host's script)"""
    def run():
        rng = np.random.default_rng(10)
        pool = _net(0).open_live_pool(**_network(rng), slots=3, window=8, timed=timed)
        totals = [9, 14, 4, 11, 7, 20, 6]
        ids, given, outs = [pool.open(100 + i) for i in range(6)], {}, []
        stalls = {1: range(3, 9), 3: range(2, 12), 5: range(5, 7)}
        for step in range(200):
            if step == 4:
                ids.append(pool.open(106))
            for j, i in enumerate(ids):
                if j in stalls and step in stalls[j]:
                    continue
                n = min(int(rng.integers(0, 3)), totals[j] - given.get(i, 0))
                if n:
                    pool.push(i, _f32(rng, CC, n) if j % 2 else torch.from_numpy(_f32(rng, CC, n)))
                    given[i] = given.get(i, 0) + n
                elif given.get(i, 0) == totals[j] and i in pool._streams and not pool._streams[i].finished:
                    pool.finish(i)
            outs.append(pool.step(audio=audio))
            if not pool._streams:
                break
        outs.append([pool.launches, pool.parks, pool.resumes])
        if timed:
            outs.append([*pool.state_seconds(), pool.prompt_seconds()])
        pool.close()
        return outs, {} if timed else None          # a timed pool reports through state_seconds and prompt_seconds
    return run


def _pool_prompts(timed):
    """prompts of 23 and 9 samples scoreable in one step, one of 14 whose frames arrive over steps, one of 40 never covered, and
    in one step four prompts for a scorer of three rows (test_live_prompt_host's scripts)"""
    def run():
        rng = np.random.default_rng(12)
        pool = _net(0).open_live_pool(**_network(rng), slots=3, window=8, fp16=True, timed=timed)
        totals = [8, 12, 6, 9, 5, 4, 4, 4, 4]
        ids = [pool.open(1), pool.open(2, _codes(rng, 23)), pool.open(3, _codes(rng, 9)), pool.open(4, _codes(rng, 14)),
               pool.open(5, _codes(rng, 40))]
        given, outs = [0] * len(totals), []
        script = {0: [2, 5, 2, 1, 2], 1: [2, 0, 0, 1, 1], 2: [2, 2, 2, 1, 2], 3: [1, 3, 2, 2, 0]}
        for step in range(80):
            if step == 6:
                ids += [pool.open(10 + P, _codes(rng, P).numpy()) for P in (4, 9, 2, 13)]
            for j, i in enumerate(ids):
                k = min(script.get(step, [2] * len(ids))[j] if j < 5 else 4, totals[j] - given[j])
                if k:
                    pool.push(i, _f32(rng, CC, k))
                    given[j] += k
                elif given[j] == totals[j] and i in pool._streams and not pool._streams[i].finished:
                    pool.finish(i)
            outs.append(pool.step(audio="int16" if step % 3 == 1 else None))
            if not pool._streams:
                break
        outs.append([pool.launches, pool.parks, pool.resumes])
        if timed:
            outs.append([*pool.state_seconds(), pool.prompt_seconds()])
        pool.close()
        return outs, {} if timed else None          # a timed pool reports through state_seconds and prompt_seconds
    return run


CASES = {
    "infer_whole_host_fp32": _infer(None, None, False, None),
    "infer_whole_philox_fp16": _infer(None, 3, True, None),
    "infer_window_host_fp16": _infer(8, None, True, None),
    "infer_window_philox_fp32": _infer(8, 3, False, None),
    "infer_prompt_window_philox": _infer(8, 3, True, 11),
    "infer_prompt_window_host": _infer(8, None, True, 11),
    "infer_prompt_on_boundary": _infer(8, 3, True, 8),
    "infer_prompt_whole_host": _infer(None, None, True, 5),
    "infer_many": _infer_many(False, False),
    "infer_many_timed": _infer_many(False, True),
    "infer_many_prompts": _infer_many(True, False),
    "infer_many_prompts_timed": _infer_many(True, True),
    "infer_many_from_features_numpy": _infer_many_from_features(False),
    "infer_many_from_features_torch": _infer_many_from_features(True),
    "log_likelihood_whole": _log_likelihood(None),
    "log_likelihood_window": _log_likelihood(8),
    "log_likelihood_from_features_whole": _log_likelihood_from_features(None, False),
    "log_likelihood_from_features_window_timed": _log_likelihood_from_features(8, True),
    "log_likelihood_many": _log_likelihood_many(False),
    "log_likelihood_many_timed": _log_likelihood_many(True),
    "log_likelihood_many_from_features": _log_likelihood_many_from_features(False),
    "log_likelihood_many_from_features_timed": _log_likelihood_many_from_features(True),
    "model_set": _model_set(False),
    "model_set_timed": _model_set(True),
    "live": _live(None, None),
    "live_int16": _live(None, "int16"),
    "live_prompt": _live(11, None),
    "live_prompt_int16": _live(6, "int16"),
    "pool_stalls": _pool_stalls(None, False),
    "pool_stalls_float_timed": _pool_stalls("float", True),
    "pool_prompts": _pool_prompts(False),
    "pool_prompts_timed": _pool_prompts(True),
}


def record(name):
    """the record of one case: its calls, its timing keys and a hash of its result"""
    global LOG
    LOG = _Log()
    try:
        with recording():
            out = CASES[name]()
        out, timing = out
        if timing is None:
            assert LOG.timing_events == 0, f"{name}: {LOG.timing_events} timing events created with timing off"
        else:
            assert LOG.timing_events > 0
        result = json.dumps(LOG.enc(out), sort_keys=True)
        return {"calls": LOG.calls, "timing": timing, "result": _hash(result.encode())}
    finally:
        LOG = None


def record_all():
    return {name: record(name) for name in CASES}


def test_serving_calls_match_the_golden_record():
    with open(GOLDEN) as f:
        golden = json.load(f)
    assert sorted(golden) == sorted(CASES)
    for name in CASES:
        got = json.loads(json.dumps(record(name)))
        want = golden[name]
        assert got["timing"] == want["timing"], name
        for k, (g, w) in enumerate(zip(got["calls"], want["calls"])):
            assert g == w, f"{name}: call {k} differs:\n got  {g}\n want {w}"
        assert len(got["calls"]) == len(want["calls"]), name
        assert got["result"] == want["result"], name
