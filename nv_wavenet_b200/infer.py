"""Host-side mirror of the reference's C++ class nvWavenetInfer<T_weight,T_data,R,S,A>
(nv_wavenet.cuh:220-640) over the C-ABI in include/nvwn_b200.h.

Same member names and argument meaning as the reference class; array arguments may be numpy
arrays (host memory) or CUDA torch tensors (device memory) -- the reference setters also accept
either kind of pointer (nv_wavenet.cuh:285-308).  All compute happens in the CUDA library.
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import FP16, FP32, FP32_FAST, KERNEL_AUTO, KERNEL_STREAM, KERNEL_TENSORCORE, MAX_MODELS, check  # noqa: F401

# Implementation enum of the reference (nv_wavenet.cuh:223-229); accepted, all map to the sm_90a kernels
AUTO, SINGLE_BLOCK, DUAL_BLOCK, PERSISTENT, MANYBLOCK_NONPERSISTENT = 0, 1, 2, 3, 4


def _model_table(what, models):
    """(void*, int32 array) of a model table, every index checked to fit a C int."""
    m = np.asarray(models, dtype=np.int64).ravel()
    if m.size and (m.min() < np.iinfo(np.int32).min or m.max() > np.iinfo(np.int32).max):
        raise ValueError(f"{what}: model indices must fit a C int; got {m.min()} .. {m.max()}")
    m = np.ascontiguousarray(m.astype(np.int32))
    return C.c_void_p(m.ctypes.data), m


def _ptr(a, dtype):
    """(void*, keepalive) of a numpy array or torch tensor holding `dtype`, C-contiguous."""
    if a is None:
        return None, None
    if isinstance(a, np.ndarray):
        if a.dtype != dtype or not a.flags["C_CONTIGUOUS"]:
            a = np.ascontiguousarray(a, dtype=dtype)
        return C.c_void_p(a.ctypes.data), a
    if hasattr(a, "data_ptr"):          # torch tensor (host or device)
        import torch
        want = torch.float32 if dtype == np.float32 else torch.int32
        if a.dtype != want or not a.is_contiguous():
            a = a.to(want).contiguous()
        return C.c_void_p(a.data_ptr()), a
    a = np.ascontiguousarray(a, dtype=dtype)
    return C.c_void_p(a.ctypes.data), a


def _stream(stream):
    if stream is None:
        return None
    if hasattr(stream, "cuda_stream"):
        return C.c_void_p(stream.cuda_stream)
    return C.c_void_p(int(stream))


def check_cond_network(num_layers, R, upsample_weight, upsample_bias, cond_weight, cond_bias, stride, error, what):
    """(C, window) of a conditioning network for num_layers layers of R residual channels: upsample_weight [C][C][window],
    upsample_bias [C], cond_weight [L*2R][C] or [L*2R][C][1], cond_bias [L*2R], and window >= stride >= 1.  Raises error(message
    naming `what`) for anything else."""
    shp = lambda a: tuple(int(v) for v in a.shape)
    lr, wu = num_layers * 2 * R, shp(upsample_weight)
    Cc = wu[0] if len(wu) == 3 and wu[0] == wu[1] else None
    if Cc is None or shp(upsample_bias) != (Cc,) or shp(cond_weight) not in ((lr, Cc), (lr, Cc, 1)) or shp(cond_bias) != (lr,):
        raise error(f"{what}: need upsample_weight [C][C][window], upsample_bias [C], cond_weight [{lr}][C] or [{lr}][C][1] and "
                    f"cond_bias [{lr}]; got {wu}, {shp(upsample_bias)}, {shp(cond_weight)}, {shp(cond_bias)}")
    if not 1 <= stride <= wu[2]:
        raise error(f"{what}: need upsampling window >= stride >= 1; got {wu[2]}, {stride}")
    return Cc, wu[2]


def split_at_wrap(first_sample, count, num_samples):
    """Absolute samples [first_sample, first_sample + count) of buffers of `num_samples` used as rings, as at most two pieces
    (position, offset, n): samples first_sample + offset .. + n - 1 sit at positions position .. position + n - 1."""
    if first_sample < 0 or count < 0 or count > num_samples:
        raise ValueError(f"need first_sample >= 0 and 0 <= count <= {num_samples}; got {first_sample}, {count}")
    pos = first_sample % num_samples
    head = min(count, num_samples - pos)
    pieces = [(pos, 0, head)] if head else []
    if head < count:
        pieces.append((0, head, count - head))
    return pieces


def live_frames(first_sample, count, window, stride):
    """Frames [lo, hi) that samples [first_sample, first_sample + count), count >= 1, of a sequence read through an upsampling
    window of `window` samples and `stride`: sample n reads frames ceil((n - window + 1) / stride) .. floor(n / stride), none below 0."""
    lo = max(0, -(-(first_sample - window + 1) // stride))
    return lo, (first_sample + count - 1) // stride + 1


def live_push_limit(frames, produced, ring_frames, window, stride):
    """The most frames a push may append to a live sequence of `frames` frames whose productions reach sample `produced`: the ring of
    `ring_frames` frames per row must keep every frame the samples from `produced` on read (nvwn_cond_producer_push)."""
    return live_frames(produced, 1, window, stride)[0] + ring_frames - frames


def live_ring_frames(samples, window, stride):
    """A ring size for live pieces of up to `samples` samples: the most frames such a piece can read, plus one for the next push,
    so every push of one frame fits once everything before it has been produced; never below ceil(window / stride) + 1."""
    return (samples + window - 2) // stride + 2


class NVWavenetInfer:
    """nvWavenetInfer(numLayers, maxDilation, batchSize, numSamples, impl=0, tanhEmbed=True)
    with the template parameters (precision, R, S, A) as keyword arguments."""

    def __init__(self, num_layers, max_dilation, batch_size, num_samples, impl=AUTO, tanh_embed=True,
                 *, R=64, S=128, A=256, dtype=FP32):
        self._l = _lib.lib()
        self.L, self.max_dilation, self.B, self.N = num_layers, max_dilation, batch_size, num_samples
        self.R, self.S, self.A, self.dtype = R, S, A, dtype
        h = C.c_void_p()
        check(self._l.nvwn_create(C.byref(h), dtype, R, S, A, num_layers, max_dilation, batch_size, num_samples,
                                  impl, int(bool(tanh_embed))), "nvwn_create")
        self._h = h
        self._samples_per_chunk = 0

    def close(self):
        if getattr(self, "_h", None):
            self._l.nvwn_destroy(self._h)
            self._h = None

    __del__ = close

    # ---- model initialisation (nv_wavenet.cuh:396-415) ----
    def set_embeddings(self, embed_prev, embed_cur):
        p, k1 = _ptr(embed_prev, np.float32); c, k2 = _ptr(embed_cur, np.float32)
        check(self._l.nvwn_set_embeddings(self._h, p, c), "setEmbeddings")

    def set_layer_weights(self, layer, Wprev, Wcur, Bh, Wres, Bres, Wskip, Bskip):
        ptrs = [_ptr(a, np.float32) for a in (Wprev, Wcur, Bh, Wres, Bres, Wskip, Bskip)]
        check(self._l.nvwn_set_layer_weights(self._h, layer, *[p for p, _ in ptrs]), "setLayerWeights")

    def set_out_weights(self, Wzs, Bzs, Wza, Bza):
        ptrs = [_ptr(a, np.float32) for a in (Wzs, Bzs, Wza, Bza)]
        check(self._l.nvwn_set_out_weights(self._h, *[p for p, _ in ptrs]), "setOutWeights")

    def load(self, w):
        """Convenience: dict with embPrev, embCur, Wprev[L], ... as produced by tests/refgen.py."""
        self.set_embeddings(w["embPrev"], w["embCur"])
        for l in range(self.L):
            self.set_layer_weights(l, w["Wprev"][l], w["Wcur"][l], w["Bh"][l], w["Wres"][l], w["Bres"][l],
                                   w["Wskip"][l], w["Bskip"][l])
        self.set_out_weights(w["Wzs"], w["Bzs"], w["Wza"], w["Bza"])

    # ---- inputs (nv_wavenet.cuh:417-422) ----
    def set_inputs(self, Lh, output_selectors):
        a, k1 = _ptr(Lh, np.float32); s, k2 = _ptr(output_selectors, np.float32)
        check(self._l.nvwn_set_inputs(self._h, a, s), "setInputs")

    def set_selectors(self, output_selectors):
        s, k = _ptr(output_selectors, np.float32)
        check(self._l.nvwn_set_selectors(self._h, s), "setSelectors")

    def set_selectors_random(self, seed, stream=None):
        """Selectors drawn on the device: counter-based (Philox-4x32-10, key = seed), see include/nvwn_b200.h."""
        check(self._l.nvwn_set_selectors_random(self._h, C.c_ulonglong(int(seed) & (2 ** 64 - 1)), _stream(stream)), "setSelectorsRandom")

    def set_conditioning(self, Lh, first_sample, num_samples, stream=None):
        a, k = _ptr(Lh, np.float32)
        check(self._l.nvwn_set_conditioning(self._h, a, first_sample, num_samples, _stream(stream)), "setConditioning")
        return k

    @staticmethod
    def _network(upsample_weight, upsample_bias, cond_weight, cond_bias):
        """((wu, bu, wc, bc) pointers, keepalive) of the four arrays of a conditioning network, as fp32."""
        pairs = [_ptr(a, np.float32) for a in (upsample_weight, upsample_bias, cond_weight, cond_bias)]
        return tuple(p for p, _ in pairs), [k for _, k in pairs]

    def _call_with_features(self, fn, name, features, upsample_weight, upsample_bias, cond_weight, cond_bias, stride, *tail):
        """fn(engine, features, C, T, upsample_weight, upsample_bias, window, stride, cond_weight, cond_bias, *tail) of the
        whole-batch producer calls, with the arrays' shapes checked; returns T * stride."""
        Cc, window = check_cond_network(self.L, self.R, upsample_weight, upsample_bias, cond_weight, cond_bias, stride, ValueError, name)
        shape = tuple(int(v) for v in features.shape)
        if len(shape) != 3 or shape[:2] != (self.B, Cc):
            raise ValueError(f"{name}: features must be [{self.B}][{Cc}][T] for this engine and network; got {shape}")
        T = shape[2]
        f, k1 = _ptr(features, np.float32)
        (wu, bu, wc, bc), keep = self._network(upsample_weight, upsample_bias, cond_weight, cond_bias)
        check(fn(self._h, f, Cc, T, wu, bu, window, stride, wc, bc, *tail), name)
        return T * stride

    def set_conditioning_from_features(self, features, upsample_weight, upsample_bias, cond_weight, cond_bias, stride,
                                       first_sample=0, stream=None):
        """Device-side WaveNet.get_cond_input (pytorch/wavenet.py:190-202) + the permutes of pytorch/nv_wavenet.py:48-49,181:
        features [B][C][T], upsample_weight [C][C][window] (ConvTranspose1d), cond_weight [L*2R][C] (or [L*2R][C][1]),
        numpy arrays or torch tensors (host or CUDA).  Fills conditioning for T*stride samples from `first_sample`."""
        return self._call_with_features(self._l.nvwn_set_conditioning_from_features, "setConditioningFromFeatures", features, upsample_weight,
                                        upsample_bias, cond_weight, cond_bias, stride, first_sample, _stream(stream))

    def cond_producer_load(self, features, upsample_weight, upsample_bias, cond_weight, cond_bias, stride, stream=None):
        """First half of set_conditioning_from_features: copies the features and both layers' weights into engine-owned device
        memory.  Returns the number of samples the sequence covers (T * stride)."""
        return self._call_with_features(self._l.nvwn_cond_producer_load, "condProducerLoad", features, upsample_weight, upsample_bias,
                                        cond_weight, cond_bias, stride, _stream(stream))

    def cond_producer_run(self, sample_begin, sample_count, first_sample=0, stream=None):
        """Second half: conditioning of samples [sample_begin, sample_begin + sample_count) of the loaded sequence, asynchronously on
        `stream` (record an event after it and make the generating stream wait for it)."""
        check(self._l.nvwn_cond_producer_run(self._h, first_sample, sample_begin, sample_count, _stream(stream)), "condProducerRun")

    def cond_producer_open_live(self, upsample_weight, upsample_bias, cond_weight, cond_bias, stride, ring_frames, stream=None):
        """Starts a live sequence of 0 frames on the whole-batch producer with the conditioning network of
        set_conditioning_from_features and a ring of `ring_frames` frames per utterance; frames then arrive with cond_producer_push
        and cond_producer_run_stream produces the samples they complete.  Replaces a loaded sequence; see nvwn_cond_producer_open_live."""
        Cc, window = check_cond_network(self.L, self.R, upsample_weight, upsample_bias, cond_weight, cond_bias, stride, ValueError,
                                        "condProducerOpenLive")
        (wu, bu, wc, bc), keep = self._network(upsample_weight, upsample_bias, cond_weight, cond_bias)
        check(self._l.nvwn_cond_producer_open_live(self._h, Cc, wu, bu, window, stride, wc, bc, ring_frames, _stream(stream)),
              "condProducerOpenLive")
        self._cond_channels = Cc

    def cond_producer_push(self, features, stream=None):
        """Appends features [B][C][n] (numpy array or torch tensor) to the live sequence.  Host frames may be reused on return; CUDA
        frames are copied in order on `stream`: keep what this returns alive until then."""
        shape = tuple(int(v) for v in features.shape)
        if len(shape) != 3 or shape[0] != self.B or shape[1] != getattr(self, "_cond_channels", shape[1]):
            raise ValueError(f"condProducerPush: features must be [{self.B}][C][n] with the C of cond_producer_open_live; got {shape}")
        f, keep = _ptr(features, np.float32)
        check(self._l.nvwn_cond_producer_push(self._h, f, shape[2], _stream(stream)), "condProducerPush")
        return keep

    # ---- streaming: the N-sample buffers used as rings (nvwn_run_stream); ranges are in absolute samples ----
    def set_selectors_random_stream(self, seed, first_sample, num_samples, stream=None):
        """Device selectors of absolute samples [first_sample, first_sample + num_samples), the values set_selectors_random gives
        an engine that holds them all."""
        check(self._l.nvwn_set_selectors_random_stream(self._h, C.c_ulonglong(int(seed) & (2 ** 64 - 1)), first_sample, num_samples,
                                                       _stream(stream)), "setSelectorsRandomStream")

    def cond_producer_run_stream(self, sample_begin, sample_count, stream=None):
        """cond_producer_run for the ring: sample s of the loaded sequence goes to position s mod N."""
        check(self._l.nvwn_cond_producer_run_stream(self._h, sample_begin, sample_count, _stream(stream)), "condProducerRunStream")

    def set_conditioning_stream(self, Lh, first_sample, stream=None):
        """Lh [n][L][B][2R]: the conditioning of absolute samples [first_sample, first_sample + n)."""
        a, k = _ptr(Lh, np.float32)
        per = self.L * self.B * 2 * self.R
        n = (k.size if isinstance(k, np.ndarray) else k.numel()) // per
        for pos, off, m in split_at_wrap(first_sample, n, self.N):
            check(self._l.nvwn_set_conditioning(self._h, C.c_void_p(a.value + off * per * 4), pos, m, _stream(stream)), "setConditioning")
        return k

    def get_yout_stream(self, out, first_sample, count, stream=None):
        """out [B][count] (numpy int32 array, or int32 torch tensor filled on `stream`) <- yOut of absolute samples
        [first_sample, first_sample + count)."""
        if isinstance(out, np.ndarray):
            stage = np.empty((self.B, self.N), np.int32)
            for pos, off, n in split_at_wrap(first_sample, count, self.N):
                self.get_yout(stage, pos, n, stream)
                out[:, off:off + n] = stage[:, pos:pos + n]
            return out
        import contextlib
        import torch
        with torch.cuda.stream(stream) if stream is not None else contextlib.nullcontext():
            stage = torch.empty((self.B, self.N), dtype=torch.int32, device=out.device)     # allocated on the stream that uses it
            for pos, off, n in split_at_wrap(first_sample, count, self.N):
                self.get_yout(stage, pos, n, stream if stream is not None else torch.cuda.current_stream())
                out[:, off:off + n].copy_(stage[:, pos:pos + n])
        return out

    def get_audio_stream(self, first_sample, count, int16=False, saturate=False, stream=None):
        """get_audio of absolute samples [first_sample, first_sample + count): numpy [B][count]."""
        pieces = [self.get_audio(pos, n, int16, saturate, stream=stream) for pos, _, n in split_at_wrap(first_sample, count, self.N)]
        return np.concatenate(pieces, axis=1) if pieces else np.empty((self.B, 0), np.int16 if int16 else np.float32)

    def run_stream(self, first_sample, count, batch_size, dump_activations=False, stream=None):
        """Generates absolute samples [first_sample, first_sample + count), count <= N, continuing from the last generation
        (first_sample 0 after reset_history).  Asynchronous on `stream`."""
        check(self._l.nvwn_run_stream(self._h, first_sample, count, batch_size, int(dump_activations), _stream(stream)), "run_stream")
        return True

    # ---- continuous batching: the B rows are slots, each restarted with a new utterance at a launch boundary ----
    def _slots(self, slots):
        """(void*, int32 array) of a list of slot or scoring-row indices."""
        s = np.ascontiguousarray(np.asarray(slots, dtype=np.int64).reshape(-1)).astype(np.int32)
        return C.c_void_p(s.ctypes.data), s

    @staticmethod
    def _seeds(what, seeds, n):
        """(void* or None, keepalive) of one uint64 seed per slot of n slots; None: no seeds (every seed 0)."""
        if seeds is None:
            return None, None
        k = np.ascontiguousarray([int(v) & (2 ** 64 - 1) for v in seeds], dtype=np.uint64)
        if k.size != n:
            raise ValueError(f"{what}: {n} slots but {k.size} seeds")
        return C.c_void_p(k.ctypes.data), k

    def restart_slots(self, slots, seeds=None, stream=None):
        """Starts a new utterance in each of `slots` at the engine's next sample: their history is cleared and silence fed back,
        the other slots are not touched.  seeds (one per slot, None = 0) key the slots' selectors for
        set_selectors_random_slots.  Asynchronous on `stream`."""
        p, s = self._slots(slots)
        k, keep = self._seeds("restart_slots", seeds, s.size)
        check(self._l.nvwn_restart_slots(self._h, p, s.size, k, _stream(stream)), "restartSlots")

    def set_conditioning_slots(self, Lh, slots, first_sample, stream=None):
        """Lh [n][L][k][2R] (numpy array or CUDA tensor): the conditioning of absolute samples [first_sample, first_sample + n)
        for the k slots `slots` only, n <= N.  A CUDA tensor is converted asynchronously on `stream` (keep it alive until then:
        it is returned)."""
        p, s = self._slots(slots)
        shape = tuple(int(v) for v in Lh.shape)
        if len(shape) != 4 or shape[1:] != (self.L, s.size, 2 * self.R):
            raise ValueError(f"set_conditioning_slots: Lh must be [n][{self.L}][{s.size}][{2 * self.R}] for {s.size} slots; got {shape}")
        a, keep = _ptr(Lh, np.float32)
        n = shape[0]
        check(self._l.nvwn_set_conditioning_slots(self._h, a, p, s.size, first_sample, n, _stream(stream)), "setConditioningSlots")
        return keep

    def set_selectors_random_slots(self, first_sample, n, stream=None):
        """Device selectors of absolute samples [first_sample, first_sample + n) for every slot from its seed and start: an
        utterance draws what a one-utterance engine draws for it."""
        check(self._l.nvwn_set_selectors_random_slots(self._h, first_sample, n, _stream(stream)), "setSelectorsRandomSlots")

    # ---- per-slot conditioning producer: each slot's conditioning from its own utterance's mel frames, on the device ----
    def cond_producer_set_weights(self, upsample_weight, upsample_bias, cond_weight, cond_bias, stride, stream=None):
        """The conditioning network of set_conditioning_from_features (upsample_weight [C][C][window], upsample_bias [C],
        cond_weight [L*2R][C] or [L*2R][C][1], cond_bias [L*2R]), for cond_producer_run_slots.  Forgets every attached utterance."""
        Cc, window = check_cond_network(self.L, self.R, upsample_weight, upsample_bias, cond_weight, cond_bias, stride, ValueError,
                                        "cond_producer_set_weights")
        (wu, bu, wc, bc), keep = self._network(upsample_weight, upsample_bias, cond_weight, cond_bias)
        check(self._l.nvwn_cond_producer_set_weights(self._h, Cc, wu, bu, window, stride, wc, bc, _stream(stream)), "condProducerSetWeights")
        self._cond_channels = Cc

    def cond_producer_set_slots(self, slots, features, starts, stream=None):
        """Attaches utterance i, mel frames features[i] [C][T_i] (numpy array or torch tensor), to slot slots[i], its sample 0 at
        absolute sample starts[i].  Host frames are copied before return; CUDA frames are copied in order on `stream`: keep what
        this returns alive until then."""
        p, s = self._slots(slots)
        if len(features) != s.size or len(starts) != s.size:
            raise ValueError(f"cond_producer_set_slots: {s.size} slots, {len(features)} frame arrays and {len(starts)} starts")
        ptrs, counts, keep = self._frames("cond_producer_set_slots", features, stream)
        st = np.ascontiguousarray([int(v) for v in starts], dtype=np.int64)
        check(self._l.nvwn_cond_producer_set_slots(self._h, p, s.size, ptrs, C.c_void_p(counts.ctypes.data), C.c_void_p(st.ctypes.data),
                                                   _stream(stream)), "condProducerSetSlots")
        return keep

    def _frames(self, what, features, stream):
        """(float*[n], int32 counts [n], keepalive) of per-slot frames [C][T_i] (numpy arrays or torch tensors; None: no frames), C
        that of cond_producer_set_weights."""
        keep, ptrs = [], (C.c_void_p * max(1, len(features)))()
        counts = np.zeros(len(features), np.int32)
        import contextlib
        on_stream = contextlib.nullcontext()
        if hasattr(stream, "cuda_stream"):                 # CUDA frames that need a contiguous fp32 copy get it on `stream`
            import torch
            on_stream = torch.cuda.stream(stream)
        with on_stream:
            for i, f in enumerate(features):
                if f is None:
                    continue
                shape = tuple(int(v) for v in f.shape)
                if len(shape) != 2 or shape[0] != getattr(self, "_cond_channels", shape[0]):
                    raise ValueError(f"{what}: frames must be [C][T] with the C of cond_producer_set_weights; got {shape}")
                a, k = _ptr(f, np.float32)
                ptrs[i], counts[i] = a, shape[1]
                keep.append(k)
        return ptrs, counts, keep

    def cond_producer_open_live_slots(self, ring_frames, stream=None):
        """Switches the per-slot producer to live mode: each slot's frames arrive over time into a ring of `ring_frames` frames
        (cond_producer_attach_live, cond_producer_push_slots), and cond_producer_run_slots produces the samples they complete.
        Forgets every attached utterance; cond_producer_set_weights and reset_history end live mode."""
        check(self._l.nvwn_cond_producer_open_live_slots(self._h, int(ring_frames), _stream(stream)), "condProducerOpenLiveSlots")

    def cond_producer_attach_live(self, slots, starts, first_frames=None, features=None, stream=None):
        """Slot slots[i] takes a live utterance whose sample 0 is absolute sample starts[i] (negative for a resumed one), holding frames
        features[i] [C][n_i] (None: none) as its frames first_frames[i] .. (None: all 0); frames before first_frames[i] count as
        pushed.  Host frames may be reused on return; CUDA frames are copied in order on `stream`: keep what this returns alive."""
        p, s = self._slots(slots)
        features = [None] * s.size if features is None else list(features)
        first = np.zeros(s.size, np.int32) if first_frames is None else np.ascontiguousarray([int(v) for v in first_frames], dtype=np.int32)
        if len(features) != s.size or len(starts) != s.size or first.size != s.size:
            raise ValueError(f"cond_producer_attach_live: {s.size} slots, {len(starts)} starts, {first.size} first frames and {len(features)} frame arrays")
        ptrs, counts, keep = self._frames("cond_producer_attach_live", features, stream)
        st = np.ascontiguousarray([int(v) for v in starts], dtype=np.int64)
        check(self._l.nvwn_cond_producer_attach_live(self._h, p, s.size, C.c_void_p(st.ctypes.data), C.c_void_p(first.ctypes.data), ptrs,
                                                     C.c_void_p(counts.ctypes.data), _stream(stream)), "condProducerAttachLive")
        return keep

    def cond_producer_push_slots(self, slots, features, stream=None):
        """Appends features[i] [C][n_i] (numpy array or torch tensor) to slot slots[i]'s live utterance.  Host frames may be reused on
        return; CUDA frames are copied in order on `stream`: keep what this returns alive until then."""
        p, s = self._slots(slots)
        if len(features) != s.size:
            raise ValueError(f"cond_producer_push_slots: {s.size} slots but {len(features)} frame arrays")
        ptrs, counts, keep = self._frames("cond_producer_push_slots", features, stream)
        check(self._l.nvwn_cond_producer_push_slots(self._h, p, s.size, ptrs, C.c_void_p(counts.ctypes.data), _stream(stream)),
              "condProducerPushSlots")
        return keep

    # ---- slot states: park a slot's utterance and resume it in any slot of a compatible engine (nvwn_save_slots) ----
    def slot_state_bytes(self):
        """Bytes of one slot state of this engine (nvwn_slot_state_bytes)."""
        n = C.c_ulonglong()
        check(self._l.nvwn_slot_state_bytes(self._h, C.byref(n)), "slotStateBytes")
        return n.value

    def save_slots(self, slots, out=None, stream=None):
        """The states of `slots` at the engine's next sample, as a uint8 CUDA tensor [n][slot_state_bytes] written asynchronously on
        `stream`, or into `out` (a uint8 CUDA tensor or numpy array of that size; a numpy array is complete on return).  The engine
        does not change."""
        p, s = self._slots(slots)
        out, ptr = self._states_out("save_slots", s.size, out)
        check(self._l.nvwn_save_slots(self._h, p, s.size, C.c_void_p(ptr), _stream(stream)), "saveSlots")
        return out

    def _states_out(self, what, n, out):
        """(out, its address) for n slot states: `out` checked as contiguous uint8 [n][slot_state_bytes], or a new CUDA tensor."""
        bytes_ = self.slot_state_bytes()
        if out is None:
            import torch
            out = torch.empty((n, bytes_), dtype=torch.uint8, device="cuda")
        size = out.size if isinstance(out, np.ndarray) else out.numel()
        contiguous = out.flags["C_CONTIGUOUS"] if isinstance(out, np.ndarray) else out.is_contiguous()
        if str(out.dtype) not in ("uint8", "torch.uint8") or size != n * bytes_ or not contiguous:
            raise ValueError(f"{what}: out must be contiguous uint8 [{n}][{bytes_}]; got {out.dtype} {tuple(out.shape)}")
        return out, out.ctypes.data if isinstance(out, np.ndarray) else out.data_ptr()

    def load_slots(self, slots, states, stream=None):
        """Slot slots[i] continues state i of `states` (uint8 [n][slot_state_bytes], numpy array or CUDA tensor, as save_slots gives
        them) from the engine's next sample.  A per-slot call; see nvwn_load_slots."""
        p, s = self._slots(slots)
        bytes_ = self.slot_state_bytes()
        if isinstance(states, np.ndarray):
            a = np.ascontiguousarray(states, dtype=np.uint8)
            ptr, size = a.ctypes.data, a.size
        else:
            a = states.contiguous()
            ptr, size = a.data_ptr(), a.numel() * a.element_size()
        if size != s.size * bytes_:
            raise ValueError(f"load_slots: {s.size} slots need {s.size} states of {bytes_} bytes; got {size} bytes")
        check(self._l.nvwn_load_slots(self._h, p, s.size, C.c_void_p(ptr), _stream(stream)), "loadSlots")
        return a

    # ---- multi-model serving (DESIGN.md §6) ----
    def set_model(self, model, src):
        """Copies the weights of engine `src` (same dtype, R, S, A, L, max_dilation and tanh_embed) into model `model`,
        1 <= model < MAX_MODELS, of this engine.  Later changes to src do not reach it; see nvwn_set_model."""
        check(self._l.nvwn_set_model(self._h, model, src._h), "setModel")

    @property
    def model_group(self):
        """Rows per model group G: rows [g*G, (g+1)*G) always run one model (nvwn_model_group)."""
        g = C.c_int()
        check(self._l.nvwn_model_group(self._h, C.byref(g)), "modelGroup")
        return g.value

    def set_group_models(self, models, stream=None):
        """The model of each of the ceil(B / model_group) groups: 0 or a model given to set_model.  Takes effect from the next
        launch on `stream`; see nvwn_set_group_models."""
        p, m = _model_table("setGroupModels", models)
        check(self._l.nvwn_set_group_models(self._h, p, m.size, _stream(stream)), "setGroupModels")

    def set_score_models(self, models, stream=None):
        """The model of each of the B scoring rows: 0 or a model given to set_model.  Applies to the scoring calls from the next one;
        ends an open scoring stream; see nvwn_set_score_models."""
        p, m = _model_table("setScoreModels", models)
        check(self._l.nvwn_set_score_models(self._h, p, m.size, _stream(stream)), "setScoreModels")

    def cond_producer_run_slots(self, slots, first_sample, num_samples, stream=None):
        """Conditioning of absolute samples [first_sample, first_sample + num_samples), num_samples <= N, for `slots` only, from
        their attached utterances (0 past an utterance's end).  Asynchronous on `stream`."""
        p, s = self._slots(slots)
        check(self._l.nvwn_cond_producer_run_slots(self._h, p, s.size, first_sample, num_samples, _stream(stream)), "condProducerRunSlots")

    def reset_history(self):
        check(self._l.nvwn_reset_history(self._h), "resetHistory")

    def set_forced(self, forced):
        f, k = _ptr(forced, np.int32)
        check(self._l.nvwn_set_forced(self._h, f), "setForced")

    # ---- fetch intermediate results (nv_wavenet.cuh:424-444) ----
    def _get(self, fn, shape, *pre):
        out = np.empty(shape, np.float32)
        check(getattr(self._l, fn)(self._h, *pre, C.c_void_p(out.ctypes.data)), fn)
        return out

    def get_xt_out(self, layer): return self._get("nvwn_get_xt_out", (self.B, self.R), layer)
    def get_skip_out(self, layer): return self._get("nvwn_get_skip_out", (self.B, self.S), layer)
    def get_zs(self): return self._get("nvwn_get_zs", (self.B, self.A))
    def get_za(self): return self._get("nvwn_get_za", (self.B, self.A))
    def get_p(self): return self._get("nvwn_get_p", (self.B, self.A))

    def activations(self):
        return {"xt": np.stack([self.get_xt_out(l) for l in range(self.L)]),
                "skip": np.stack([self.get_skip_out(l) for l in range(self.L)]),
                "zs": self.get_zs(), "za": self.get_za(), "p": self.get_p()}

    def get_yout(self, y_out, offset, size, stream=None):
        p, k = _ptr(y_out, np.int32)
        check(self._l.nvwn_get_yout(self._h, p, offset, size, _stream(stream)), "getYOut")

    def get_audio(self, offset=0, size=None, int16=False, saturate=False, out=None, stream=None):
        """Device-side replacement of the reference's host post-processing (pytorch/nv_wavenet_inference.py:55-60):
        mu-law decode (utils.mu_law_decode_numpy, mu_quantization = A) of yOut[:, offset:offset+size], as float32
        in [-1, 1] or, with int16=True, as `(MAX_WAV_VALUE * audio).astype('int16')`.  `out`: numpy array or torch
        tensor [B][size] of the matching dtype (a CUDA tensor is filled asynchronously on `stream`); allocated
        (numpy) if None.  saturate=False keeps the reference's cast of the top code (+1.0 -> -32768)."""
        size = self.N - offset if size is None else size
        if out is None:
            out = np.empty((self.B, size), np.int16 if int16 else np.float32)
        if isinstance(out, np.ndarray):
            ok = out.flags["C_CONTIGUOUS"] and out.dtype == (np.int16 if int16 else np.float32) and out.size == self.B * size
            p = C.c_void_p(out.ctypes.data)
        else:                               # torch tensor
            import torch
            ok = out.is_contiguous() and out.dtype == (torch.int16 if int16 else torch.float32) and out.numel() == self.B * size
            p = C.c_void_p(out.data_ptr())
        if not ok:                          # the library writes B * size values into it
            raise ValueError(f"get_audio: out must be contiguous {'int16' if int16 else 'float32'} [{self.B}][{size}]; got "
                             f"{out.dtype} {tuple(out.shape)}")
        check(self._l.nvwn_get_audio(self._h, None if int16 else p, p if int16 else None, offset, size, int(saturate),
                                     _stream(stream)), "getAudio")
        return out

    # ---- teacher-forced scoring (nvwn_score) ----
    def score(self, audio, num_samples=None, batch_size=None, logits=False, stream=None):
        """Log-likelihood of given audio under the engine's fp16 model: logp[b][t] = log softmax(Za_t)[audio[b][t]], with
        audio[b][0..t) fed back and the conditioning already in the engine.  `audio`: int [batch][samples] numpy array
        (numpy results) or CUDA tensor (CUDA tensors, filled asynchronously on `stream`).  Returns logp [batch_size][num_samples],
        or (logp, logits [batch_size][num_samples][A]) with logits=True.  The generation state is left untouched."""
        return self._score(audio, num_samples, batch_size, logits, "score",
                           lambda a, n, bs, lp, lg: self._l.nvwn_score(self._h, a, n, bs, lp, lg, _stream(stream)))

    def score_stream(self, audio, first_sample, num_samples=None, batch_size=None, logits=False, stream=None):
        """Scoring of audio of any length through this engine, a window at a time: the log-likelihood of absolute samples
        [first_sample, first_sample + num_samples), num_samples <= N, continuing the scoring stream (first_sample 0 starts one).
        `audio` holds this call's samples only, [batch][num_samples], and sample t uses the conditioning at position t mod N.
        Arrays and results as for score().  Over the windows the results equal score() of one engine of the whole length."""
        return self._score(audio, num_samples, batch_size, logits, "score_stream",
                           lambda a, n, bs, lp, lg: self._l.nvwn_score_stream(self._h, a, first_sample, n, bs, lp, lg, _stream(stream)))

    def score_stream_packed(self, audio, starts, first_sample, num_samples=None, batch_size=None, logits=False, stream=None):
        """score_stream of a queue of utterances packed end to end in the rows: starts [batch][num_samples] (numpy array or CUDA
        tensor), nonzero where a new utterance begins in that row at that sample.  From its start each utterance's results are the
        bits score() gives it alone on the same conditioning.  first_sample 0 opens a packed stream (every row starts there); a
        packed stream is continued only by this call.  Arrays and results as for score(); see nvwn_score_stream_packed."""
        n = audio.shape[1] if num_samples is None else num_samples
        bs = audio.shape[0] if batch_size is None else batch_size
        shape = tuple(int(v) for v in starts.shape)
        if len(shape) != 2 or shape[0] < bs or shape[1] < n:
            raise ValueError(f"score_stream_packed: starts must be [batch][samples] covering [{bs}][{n}]; got {shape}")
        if hasattr(starts, "is_cuda") and starts.is_cuda:
            import torch
            flags = (starts[:bs, :n] != 0).to(torch.uint8).contiguous()
            p = flags.data_ptr()
        else:
            flags = np.ascontiguousarray(np.asarray(starts)[:bs, :n] != 0, dtype=np.uint8)
            p = flags.ctypes.data
        return self._score(audio, n, bs, logits, "score_stream_packed",
                           lambda a, n, bs, lp, lg: self._l.nvwn_score_stream_packed(self._h, a, C.c_void_p(p), first_sample, n, bs, lp, lg,
                                                                                     _stream(stream)))

    def prime_from_score(self, stream=None):
        """After score_stream over a prompt, samples [0, P): generation continues the prompt from sample P, run_stream(P, count, bs)
        with the scoring stream's batch_size bs.  The scoring stream stays open.  Asynchronous on `stream`; see nvwn_prime_from_score."""
        check(self._l.nvwn_prime_from_score(self._h, _stream(stream)), "primeFromScore")

    def prime_slots_from_score(self, rows, slots, seeds=None, stream=None):
        """After score_stream over prompts [0, P): slot slots[i] starts an utterance whose samples [0, P) are scoring row rows[i],
        continued by generation from the engine's next sample t0 (its sample P at t0).  seeds (one per slot, None = 0) key the slots'
        selectors as restart_slots does.  The scoring stream stays open.  Asynchronous on `stream`; see nvwn_prime_slots_from_score."""
        p, s = self._slots(slots)
        pr, r = self._slots(rows)
        if r.size != s.size:
            raise ValueError(f"prime_slots_from_score: {s.size} slots but {r.size} rows")
        k, keep = self._seeds("prime_slots_from_score", seeds, s.size)
        check(self._l.nvwn_prime_slots_from_score(self._h, pr, p, s.size, k, _stream(stream)), "primeSlotsFromScore")

    def score_save_states(self, rows, seeds=None, out=None, stream=None):
        """After score_stream over prompts [0, P): the slot states of scoring rows `rows` at P, as a uint8 CUDA tensor
        [n][slot_state_bytes] written asynchronously on `stream`, or into `out` as for save_slots; seeds (one per row, None = 0) are
        the states' selector keys.  load_slots resumes them in any slot of a compatible engine.  The scoring stream stays open; see
        nvwn_score_save_states."""
        pr, r = self._slots(rows)
        k, keep = self._seeds("score_save_states", seeds, r.size)
        out, ptr = self._states_out("score_save_states", r.size, out)
        check(self._l.nvwn_score_save_states(self._h, pr, r.size, k, C.c_void_p(ptr), _stream(stream)),
              "scoreSaveStates")
        return out

    def _score(self, audio, num_samples, batch_size, logits, what, call):
        """audio[:batch_size, :num_samples] as int32 and the outputs of score() in matching memory; call(audio, n, bs, logp, logits)
        with their pointers."""
        n = audio.shape[1] if num_samples is None else num_samples
        bs = audio.shape[0] if batch_size is None else batch_size
        if hasattr(audio, "is_cuda") and audio.is_cuda:
            import torch
            a = audio[:bs, :n].to(torch.int32).contiguous()
            lp = torch.empty((bs, n), dtype=torch.float32, device=audio.device)
            lg = torch.empty((bs, n, self.A), dtype=torch.float32, device=audio.device) if logits else None
            ptrs = (a.data_ptr(), lp.data_ptr(), lg.data_ptr() if logits else None)
        else:
            a = np.ascontiguousarray(np.asarray(audio)[:bs, :n], dtype=np.int32)
            lp = np.empty((bs, n), np.float32)
            lg = np.empty((bs, n, self.A), np.float32) if logits else None
            ptrs = (a.ctypes.data, lp.ctypes.data, lg.ctypes.data if logits else None)
        check(call(C.c_void_p(ptrs[0]), n, bs, C.c_void_p(ptrs[1]), None if ptrs[2] is None else C.c_void_p(ptrs[2])), what)
        return (lp, lg) if logits else lp

    # ---- run (nv_wavenet.cuh:445-639) ----
    def run_partial(self, init_sample, num_samples, batch_size, y_out=None, batch_size_per_block=1,
                    dump_activations=False, stream=None):
        count = self._samples_per_chunk if self._samples_per_chunk else num_samples
        p, k = _ptr(y_out, np.int32)
        check(self._l.nvwn_run_partial(self._h, init_sample, count, num_samples, batch_size, p,
                                       int(dump_activations), _stream(stream)), "run_partial")
        return True

    def run(self, num_samples, batch_size, y_out=None, batch_size_per_block=1, dump_activations=False, stream=None):
        """Returns True like the reference; y_out (numpy int32 [B][N] or CUDA int tensor) is filled
        asynchronously on `stream` exactly as the reference does -- synchronize() before reading."""
        self._samples_per_chunk = 0
        return self.run_partial(0, num_samples, batch_size, y_out, batch_size_per_block, dump_activations, stream)

    def run_chunks(self, num_samples_per_chunk, consume, num_samples, batch_size, y_out=None,
                   batch_size_per_block=1, dump_activations=False, stream=None):
        """run_chunks (nv_wavenet.cuh:445-497): launch chunk after chunk; each chunk of yOut is copied
        out on a second stream as soon as it is produced; consume(yOut, initSample, count) per chunk."""
        import torch
        compute = stream if stream is not None else torch.cuda.current_stream()
        copy = torch.cuda.Stream()
        chunks = []
        for init in range(0, num_samples, num_samples_per_chunk):
            n = min(num_samples_per_chunk, num_samples - init)
            self._samples_per_chunk = n
            self.run_partial(init, num_samples, batch_size, None, batch_size_per_block, True, compute)
            ev = torch.cuda.Event(); ev.record(compute)
            copy.wait_event(ev)
            if y_out is not None:
                self.get_yout(y_out, init, n, copy)
            done = torch.cuda.Event(); done.record(copy)
            chunks.append((init, n, done))
        self._samples_per_chunk = 0
        for init, n, done in chunks:
            done.synchronize()
            consume(y_out, init, n)
        return True

    def synchronize(self):
        import torch
        torch.cuda.synchronize()

    def launch_info(self):
        info = _lib.LaunchInfo()
        check(self._l.nvwn_get_launch_info(self._h, C.byref(info)), "launch_info")
        return {k: getattr(info, k) for k, _ in _lib.LaunchInfo._fields_}

    def weight_blob(self):
        p = C.c_void_p(); n = C.c_ulonglong()
        check(self._l.nvwn_weight_blob(self._h, C.byref(p), C.byref(n)), "weight_blob")
        return p.value, n.value

    def weights_updated(self):
        check(self._l.nvwn_weights_updated(self._h), "weights_updated")
