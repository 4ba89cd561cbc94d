"""PyTorch-facing binding with the surface of the reference's `pytorch/nv_wavenet.py` -- class `NVWaveNet`, the `Impl`
constants and `column_major` -- implemented over the handle C-ABI (include/nvwn_b200.h) through ctypes (the reference's
THC-era pybind wrapper, `pytorch/wavenet_infer_wrapper.cpp`, no longer builds against torch >= 2).

    wavenet = NVWaveNet(**model.export_weights())
    samples = wavenet.infer(cond_input, Impl.PERSISTENT)      # int32 CUDA tensor [batch, samples]

Unlike the reference wrapper (pytorch/wavenet_infer.cu:87-145 builds the whole nvWavenetInfer object, uploads every weight and
frees it again on EVERY call) the object keeps a persistent engine per (batch, samples, precision): weights are uploaded once,
infer() only sets the inputs.  Selectors: `seed=None` draws them like the reference (libc rand(), replayable with srand());
an integer seed draws them on the device (counter-based Philox, include/nvwn_b200.h).

Constructor arguments, accepted shapes, the appended unused residual layer and the memory layouts handed to the
kernel are those of pytorch/nv_wavenet.py:55-196; the code is organised around one table of expected shapes.
"""
import ctypes as C
from collections import deque

import numpy as np
import torch

from . import _lib
from .infer import check_cond_network, live_frames, live_push_limit, live_ring_frames


class Impl:
    """`implementation` argument of infer() (pytorch/nv_wavenet.py:51-54); one kernel family serves all of them here."""
    AUTO = 0
    SINGLE_BLOCK = 1
    DUAL_BLOCK = 2
    PERSISTENT = 3


def column_major(x):
    """Row-major torch tensor -> the column-major layout the kernel reads (pytorch/nv_wavenet.py:33-49):
    vectors unchanged, [M][K] and conv-style [M][K][1] matrices transposed, 4-D conditioning fully reversed."""
    nd = x.dim()
    if nd == 1:
        return x
    if nd == 3:
        if x.size(2) != 1:
            raise AssertionError("column_major: 3-D tensors must be convolution weights of kernel size 1")
        x, nd = x[:, :, 0], 2
    if nd == 2:
        return x.t().contiguous()
    if nd == 4:
        return x.permute(3, 2, 1, 0).contiguous()
    raise AssertionError(f"column_major: unsupported rank {nd}")


def plan_slots(lengths, slots, window, models=None, group=1):
    """Continuous batching schedule of infer_many: utterances of `lengths` samples, in arrival order, through `slots` slots
    restarted only at multiples of `window`.  At each window boundary the free slots (lowest first) take the next queued
    utterances; a slot is free once its utterance has ended.  Returns [(slot, start)] per utterance, start a multiple of window.
    models: None, or the model of each utterance (ModelSet.infer_many), slots in groups of `group` that run one model at a time
    (slots [g*group, (g+1)*group)): a free slot takes the earliest queued utterance whose model its group runs, and a group with
    no live utterance first takes the model of the earliest queued one.  A group so runs one model for every utterance's whole
    span.  models=None is the one-model schedule."""
    if slots < 1 or window < 1 or group < 1:
        raise ValueError(f"need slots >= 1, window >= 1 and group >= 1; got {slots}, {window}, {group}")
    if any(n < 1 for n in lengths):
        raise ValueError("every utterance needs at least one sample")
    if models is None:
        models = [0] * len(lengths)
    elif len(models) != len(lengths) or any(int(m) != m or m < 0 for m in models):
        raise ValueError(f"need one model index >= 0 per utterance; got {len(models)} for {len(lengths)} utterances")
    ends = [0] * slots                              # sample at which each slot's current utterance ends
    runs = [None] * ((slots + group - 1) // group)  # the model each group runs while it has a live utterance
    waiting = {}                                    # model -> its queued utterances, in arrival order
    for u, m in enumerate(models):
        waiting.setdefault(m, deque()).append(u)
    plan, left, t = [None] * len(lengths), len(lengths), 0
    while left:
        for s in range(slots):
            if ends[s] > t or not left:
                continue
            g = s // group
            if all(ends[x] <= t for x in range(g * group, min(slots, (g + 1) * group))):
                runs[g] = models[min(q[0] for q in waiting.values())]
            q = waiting.get(runs[g])
            if q:
                u = q.popleft()
                if not q:
                    del waiting[runs[g]]
                plan[u] = (s, t)
                ends[s] = t + lengths[u]
                left -= 1
        if left:
            t = (min(e for e in ends if e > t) + window - 1) // window * window   # the next boundary at which a slot is free
    return plan


def _reset(eng):
    """eng.reset_history(), which writes on the default stream, with the current stream ordered after it"""
    eng.reset_history()
    torch.cuda.current_stream().wait_stream(torch.cuda.default_stream())


def _windows(plan, lengths, window):
    """The windows of a plan_slots schedule: per window, (first sample, samples, utterances that start there, live slots as
    [(slot, utterance, its first sample in the window, its samples in the window)], slots ascending)."""
    end = max((start + n for (_, start), n in zip(plan, lengths)), default=0)
    by_start = {}
    for u, (s, start) in enumerate(plan):
        by_start.setdefault(start, []).append(u)
    active, out = {}, []                                           # slot -> utterance
    for first in range(0, end, window):
        count = min(window, end - first)
        starting = by_start.get(first, [])
        for u in starting:
            active[plan[u][0]] = u
        live = [(s, u, first - plan[u][1], min(count, plan[u][1] + lengths[u] - first))
                for s, u in sorted(active.items()) if plan[u][1] + lengths[u] > first]
        out.append((first, count, starting, live))
    return out


def plan_packed(lengths, slots):
    """Packed scoring schedule of log_likelihood_many: utterances of `lengths` samples, in arrival order, each to the row whose
    current end is earliest (the lowest row on ties), starting at that end.  Returns [(slot, start)] per utterance."""
    if slots < 1:
        raise ValueError(f"need slots >= 1; got {slots}")
    if any(n < 1 for n in lengths):
        raise ValueError("every utterance needs at least one sample")
    ends, plan = [0] * slots, []
    for n in lengths:
        s = ends.index(min(ends))
        plan.append((s, ends[s]))
        ends[s] += n
    return plan


def plan_packed_models(lengths, models, slots):
    """Packed scoring schedule of ModelSet.log_likelihood_many: utterances of `lengths` samples, utterance u scored with model
    models[u], through `slots` rows that each keep one model.  The rows are split among the distinct models, in model order, in
    proportion to their total samples: each gets 1 + floor((slots - V) * share) rows, V distinct models, and the rows left over
    go to the model of most samples (the lowest on ties).  Within a model's rows its utterances, in arrival order, follow
    plan_packed.  Returns (plan, table): [(row, start)] per utterance, and the model of each row."""
    if len(models) != len(lengths) or any(int(m) != m or m < 0 for m in models):
        raise ValueError(f"need one model index >= 0 per utterance; got {len(models)} for {len(lengths)} utterances")
    if any(n < 1 for n in lengths):
        raise ValueError("every utterance needs at least one sample")
    totals = {}
    for n, m in zip(lengths, models):
        totals[int(m)] = totals.get(int(m), 0) + n
    used = sorted(totals)
    if slots < len(used):
        raise ValueError(f"{len(used)} distinct models need at least as many slots; got {slots}")
    whole = sum(totals.values())
    rows = {m: 1 + (slots - len(used)) * totals[m] // whole for m in used}
    rows[max(used, key=lambda m: (totals[m], -m))] += slots - sum(rows.values())
    plan, table, base = [None] * len(lengths), [], 0
    for m in used:
        mine = [u for u in range(len(lengths)) if models[u] == m]
        for u, (s, start) in zip(mine, plan_packed([lengths[u] for u in mine], rows[m])):
            plan[u] = (base + s, start)
        table += [m] * rows[m]
        base += rows[m]
    return plan, table


def _packed_windows(plan, lengths, window):
    """The windows of a plan_packed schedule at multiples of `window`: per window (first sample, samples, segments), a segment
    (slot, utterance, its first sample in the utterance, its first sample in the window, samples) for every utterance that has
    samples in the window, ordered by slot and, within a slot, by time."""
    rows = {}
    for u, (s, _) in enumerate(plan):
        rows.setdefault(s, []).append(u)                          # in arrival order, which is time order within a row
    end = max((start + n for (_, start), n in zip(plan, lengths)), default=0)
    done = {s: 0 for s in rows}                                   # per row, its utterances that ended before the window
    out = []
    for first in range(0, end, window):
        last = min(first + window, end)
        segs = []
        for s in sorted(rows):
            us, i = rows[s], done[s]
            while i < len(us) and plan[us[i]][1] + lengths[us[i]] <= first:
                i += 1
            done[s] = i
            while i < len(us) and plan[us[i]][1] < last:
                u, start = us[i], plan[us[i]][1]
                b, e = max(start, first), min(start + lengths[u], last)
                segs.append((s, u, b - start, b - first, e - b))
                i += 1
        out.append((first, last - first, segs))
    return out


def _pack_window(count, segs, audios, slots):
    """The audio [slots][count] (int32, code 128 where a row has no utterance) and start flags [slots][count] (uint8, 1 at each
    utterance's first sample) of one window's segments (_packed_windows), on the device of `audios`, per utterance int32 [n_u]."""
    dev = audios[0].device if audios else "cpu"
    audio = torch.full((slots, count), 128, dtype=torch.int32, device=dev)
    rows, cols = [], []
    for s, u, a, o, m in segs:
        audio[s, o:o + m] = audios[u][a:a + m]
        if a == 0:
            rows.append(s)
            cols.append(o)
    starts = torch.zeros((slots, count), dtype=torch.uint8, device=dev)
    starts[torch.tensor(rows, dtype=torch.long, device=dev), torch.tensor(cols, dtype=torch.long, device=dev)] = 1
    return audio, starts


def _expect(name, tensor, shape):
    got = tuple(tensor.size())[:len(shape)]
    if got != tuple(shape):
        raise AssertionError(f"{name}: shape {got} does not match the compiled kernel's {tuple(shape)}")


def _check_window(window):
    if window is not None and window < 1:
        raise AssertionError(f"window must be at least 1; got {window}")


def _check_rows(what, name, rows, window):
    """The rows (`name`: slots or batch_size) and window of an engine a call makes: both at least 1."""
    if rows < 1 or window is None or window < 1:
        raise AssertionError(f"{what}: need {name} >= 1 and window >= 1; got {rows}, {window}")


def _check_frames(features, C):
    """The frame counts T_u of per-utterance mel frames [C][T_u], each T_u >= 1."""
    shapes = [tuple(int(v) for v in f.shape) for f in features]
    for s in shapes:
        if len(s) != 2 or s[0] != C or s[1] < 1:
            raise AssertionError(f"each utterance's frames are [{C}][T] with T >= 1; got {s}")
    return [s[1] for s in shapes]


class _Timer:
    """GPU time between named points of the work on a stream, for a `timing` dict (None: timing is off).  mark(name, stream)
    records an event there when timing is on and does nothing (no event) when it is off; seconds(start, end) sums, over the marks
    in order, the time from the i-th `start` mark to the i-th `end` mark; report(key=(start, end), ...) puts those sums into the
    dict.  Read it after a synchronise."""

    def __init__(self, timing):
        self.on, self.timing, self._marks = timing is not None, timing, {}

    def mark(self, name, stream=None):
        if self.on:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record(stream)
            self._marks.setdefault(name, []).append(ev)

    def seconds(self, start, end):
        return sum(a.elapsed_time(b) for a, b in zip(self._marks.get(start, ()), self._marks.get(end, ()))) / 1e3

    def report(self, **spans):
        if self.on:
            self.timing.update({key: self.seconds(start, end) for key, (start, end) in spans.items()})


def _score_prompt_group(eng, prompts, fill, at_end, **stream):
    """One scoring stream on `eng` (W = eng.N samples) whose row j is prompts[j], int32 codes [P_j] on the device, rows by length.
    It is scored in pieces that end at each distinct P_j and at multiples of W, each after fill(a, m) has put the conditioning of
    samples [a, a + m) into the store; a row past its prompt's end is scored on code 128 and its results are unused.  At each
    distinct P, at_end(rows) acts on the rows whose prompt ends there.  stream: stream=s to score on s, or nothing."""
    ends = [int(p.numel()) for p in prompts]
    codes = torch.full((len(prompts), ends[-1]), 128, dtype=torch.int32, device=prompts[0].device)
    for j, p in enumerate(prompts):
        codes[j, :ends[j]] = p
    a, W = 0, eng.N
    for end in sorted(set(ends)):
        while a < end:
            m = min(end - a, W - a % W)
            fill(a, m)
            eng.score_stream(codes[:, a:a + m], a, **stream)
            a += m
        at_end([j for j, P in enumerate(ends) if P == end])


def _score_windows(windows, fill, score, timing):
    """The window loop of the log_likelihood family: per window w, fill(*w) puts its conditioning into the store and score(*w)
    scores it; then a synchronise.  timing: None, or a dict for the GPU seconds of fill ("produce_s") and of scoring ("score_s")."""
    timer = _Timer(timing)
    for w in windows:
        timer.mark("fill")
        fill(*w)
        timer.mark("score")
        score(*w)
        timer.mark("done")
    torch.cuda.synchronize()
    timer.report(produce_s=("fill", "score"), score_s=("score", "done"))


def _score_then_generate(eng, prompt, first, m, select, read):
    """Samples [first, first + m) of a batch on `eng`, their conditioning already in the store: with a prompt [batch][P], the part
    before P is scored and the engine primed at P; the rest, [g0, g0 + k), gets its selectors from select(g0, k), is generated
    and read out by read(g0, k)."""
    P, g0 = 0 if prompt is None else prompt.shape[1], first
    if first < P:
        g0 = min(first + m, P)
        eng.score_stream(prompt[:, first:g0], first)
        if g0 == P:
            eng.prime_from_score()
    k = first + m - g0
    if k:
        select(g0, k)
        eng.run_stream(g0, k, eng.B)
        read(g0, k)


def check_prompt(what, prompt, rows, n, fp16, A):
    """Checks a prompt: int mu-law codes [P] (rows None) or [rows][P], 1 <= P < n (n None: no upper bound), each in [0, A), with
    fp16 set, since prompts are scored by the fp16 scorer.  Returns it as a tensor."""
    p = torch.as_tensor(prompt)
    lead = () if rows is None else (rows,)
    shape = tuple(p.shape)
    if len(shape) != len(lead) + 1 or shape[:-1] != lead or not 1 <= shape[-1] or (n is not None and shape[-1] >= n):
        bound = "1 <= P" if n is None else f"1 <= P < {n}"
        raise AssertionError(f"{what} must be {''.join(f'[{r}]' for r in lead)}[P] with {bound}; got {shape}")
    if p.dtype.is_floating_point or p.dtype.is_complex or p.dtype == torch.bool:
        raise AssertionError(f"{what} must hold integer mu-law codes; got {p.dtype}")
    if int(p.min()) < 0 or int(p.max()) >= A:
        raise AssertionError(f"{what} holds codes outside [0, {A})")
    if not fp16:
        raise AssertionError(f"{what} needs fp16=True: prompts are scored by the fp16 scorer")
    return p


def prompt_frames(P, stride):
    """The frames a prompt of P samples needs before it can be scored: samples [0, P) read frames up to floor((P - 1) / stride)."""
    return (P - 1) // stride + 1


def plan_prompt_groups(prompted, rows):
    """The scoring streams of one LivePool.step: the streams in `prompted` [(id, P)], in order, in groups of at most `rows` (the
    scoring engine's rows), each group's rows by prompt length.  Returns [[(id, P)] per group]; row j of a group is its j-th entry."""
    return [sorted(prompted[k:k + rows], key=lambda x: x[1]) for k in range(0, len(prompted), rows)]


class LiveSession:
    """Live vocoding of one batch of utterances whose mel frames arrive over time (NVWaveNet.open_live): each push appends frames
    and generates every sample they complete, so audio starts with the first frames and an open-ended stream can be vocoded.
    The session owns its engine of `window` samples; close() releases it.
    With a prompt [batch][P] (int32 CUDA codes), the frames' first P samples are not generated: as the pushes complete them they
    are scored on the session's engine (nvwn_score_stream), which then continues the prompt from sample P (nvwn_prime_from_score)."""

    device = "cuda"                 # where push() puts its samples

    def __init__(self, eng, channels, upsample_window, stride, seed, window, prompt=None):
        self._eng = eng
        self.channels, self.upsample_window, self.stride, self.seed, self.window = channels, upsample_window, stride, seed, window
        self.ring_frames = live_ring_frames(window, upsample_window, stride)
        self.prompt = prompt
        self.frames = 0             # frames pushed so far
        self.samples = 0            # samples scored or generated so far: every sample the frames complete, [0, frames * stride)

    def push(self, frames, audio=None, saturate=False):
        """Appends frames [batch][C][n] (numpy array or torch tensor, n >= 0) and generates samples [samples, (frames + n) * stride),
        in pieces of at most `window` samples, each one's conditioning produced from the ring just before it is generated.  Frames
        the ring cannot take at once are fed in pieces, each generated before the next is pushed.  Returns those samples as an
        int32 CUDA tensor [batch][k]; with audio="float" or "int16" returns (samples, audio), audio the mu-law decoded samples
        [batch][k] as a numpy array (get_audio_stream; saturate as for get_audio).  Together the pushes give infer() of the finished
        utterance with the same seed and window, bit for bit.  With a prompt of P samples, samples before P are scored instead and
        not returned: the pushes give infer(prompt=prompt)[:, P:]."""
        if audio not in (None, "float", "int16"):
            raise AssertionError(f"push: audio is None, 'float' or 'int16'; got {audio!r}")
        shape = tuple(int(v) for v in frames.shape)
        if len(shape) != 3 or shape[:2] != (self._eng.B, self.channels):
            raise AssertionError(f"push: frames must be [{self._eng.B}][{self.channels}][n]; got {shape}")
        frames = frames.to(torch.float32) if isinstance(frames, torch.Tensor) else np.asarray(frames, np.float32)
        eng, n, done = self._eng, shape[2], 0
        ys, auds = [], []

        def read(first, m):
            ys.append(eng.get_yout_stream(torch.empty((eng.B, m), dtype=torch.int32, device=self.device), first, m))
            if audio is not None:
                auds.append(eng.get_audio_stream(first, m, int16=audio == "int16", saturate=saturate))

        while True:
            k = min(n - done, live_push_limit(self.frames, self.samples, self.ring_frames, self.upsample_window, self.stride))
            if k > 0:
                eng.cond_producer_push(frames[:, :, done:done + k])
                self.frames += k
                done += k
            end = self.frames * self.stride
            P = 0 if self.prompt is None else self.prompt.shape[1]
            while self.samples < end:
                first, m = self.samples, min(self.window, end - self.samples)
                if first < P:
                    m = min(m, P - first)                         # a piece is all prompt or all generated
                eng.cond_producer_run_stream(first, m)
                _score_then_generate(eng, self.prompt, first, m, lambda g0, k: eng.set_selectors_random_stream(self.seed, g0, k), read)
                self.samples += m
            if done == n:
                break
        y = torch.cat(ys, dim=1) if ys else torch.empty((eng.B, 0), dtype=torch.int32, device=self.device)
        if audio is None:
            return y
        return y, np.concatenate(auds, axis=1) if auds else np.empty((eng.B, 0), np.int16 if audio == "int16" else np.float32)

    def close(self):
        if self._eng is not None:
            self._eng.close()
            self._eng = None


def live_ready(position, frames, finished, window, stride):
    """Whether a live stream can take a launch of `window` samples: its `frames` frames complete at least `window` samples past the
    `position` it has generated, or it is finished and has samples left."""
    return frames * stride - position >= window or (finished and frames * stride > position)


def plan_live_step(resident, waiting, slots, window, stride):
    """The slot decision of one LivePool.step, from the streams' counters alone.  resident: {id: (slot, position, frames, finished)}
    of the streams in slots; waiting: [(id, position, frames, finished)] of the others, in the order they began to wait.  Resident
    streams that are not ready (live_ready) are parked; ready waiting streams take the free slots (lowest first) in FIFO order.
    Returns (parked ids, [(id, slot)] of the streams that take a slot)."""
    park = [i for i, (_, p, f, fin) in resident.items() if not live_ready(p, f, fin, window, stride)]
    held = {s for i, (s, _, _, _) in resident.items() if i not in park}
    free = [s for s in range(slots) if s not in held]
    place = []
    for i, p, f, fin in waiting:
        if free and live_ready(p, f, fin, window, stride):
            place.append((i, free.pop(0)))
    return park, place


class _LiveStream:
    """A LivePool stream's counters and its frames on the host: frames [base, base + held) of the `frames` given so far, `pushed` of
    them in its slot's ring while it is resident, the samples it has generated (`position`), and its state while parked."""

    def __init__(self, seed, channels, prompt=None):
        self.seed, self.finished, self.prompt = seed, False, prompt          # prompt: int32 CUDA [P] until it is scored, then None
        self.buf, self.base, self.frames = np.empty((channels, 64), np.float32), 0, 0
        self.position, self.slot, self.pushed, self.state, self.started = 0, None, 0, None, False

    def append(self, frames):
        n = frames.shape[1]
        held = self.frames - self.base
        if held + n > self.buf.shape[1]:
            grown = np.empty((self.buf.shape[0], max(2 * self.buf.shape[1], held + n)), np.float32)
            grown[:, :held] = self.buf[:, :held]
            self.buf = grown
        self.buf[:, held:held + n] = frames
        self.frames += n

    def span(self, lo, hi):
        """frames [lo, hi) as [C][hi - lo]"""
        return self.buf[:, lo - self.base:hi - self.base]

    def drop_before(self, lo):
        """forgets the frames before lo"""
        if lo > self.base:
            held = self.frames - lo
            self.buf[:, :held] = self.buf[:, lo - self.base:self.frames - self.base].copy()
            self.base = lo


class LivePool:
    """Live serving: many live streams, each with its own mel frames arriving at its own pace, share one engine of `slots` rows and
    `window` samples (NVWaveNet.open_live_pool).  push() only stores frames; each step() generates one window for the streams whose
    frames complete it.  A stream whose frames are late is parked: its slot state is saved (nvwn_save_slots) and its slot given to a
    stream that is ready; once its frames arrive it is loaded into any free slot (nvwn_load_slots) and goes on with the bits it
    would have had without the pause.  So stream s's outputs, concatenated, equal infer() of its finished frames' conditioning with
    its seed, bit for bit, however its frames were paced.  The pool owns its engine; close() releases it.
    A stream opened with a prompt continues given audio: once its frames cover the prompt, the prompt is scored on a scoring engine
    the pool owns and its state saved there (nvwn_score_save_states); the stream then waits as a parked stream at position P and is
    resumed like one.  Its outputs are infer(cond, seed=seed, fp16=True, prompt=prompt)[0, P:], bit for bit."""

    device = "cuda"                 # where step() puts its samples

    def __init__(self, eng, channels, upsample_window, stride, timed=False, scorer=None, network=None):
        """eng: an engine whose per-slot producer has the conditioning network (cond_producer_set_weights); the pool opens its live
        mode, with rings of live_ring_frames(N, upsample_window, stride) frames.  timed: record the GPU time of saves, loads and
        prompt scoring.  scorer: None (no prompts), or a callable that makes the pool's scoring engine, an fp16 engine with eng's
        weights, called when the first prompt is scored; network: the conditioning network (upsample_weight, upsample_bias,
        cond_weight [L*2R][C], cond_bias) for its whole-batch producer."""
        self._eng = eng
        self._scorer, self._scorer_eng, self._network = scorer, None, network
        self.channels, self.upsample_window, self.stride, self.window = channels, upsample_window, stride, eng.N
        self.ring_frames = live_ring_frames(self.window, upsample_window, stride)
        eng.cond_producer_open_live_slots(self.ring_frames)
        self.t = 0                                      # the engine's next sample
        self.launches = self.parks = self.resumes = 0
        self._streams, self._waiting, self._next_id = {}, [], 0
        self._stage = None                              # yOut staging [B][N], allocated on the first launch
        self._timer = _Timer({} if timed else None)         # read by state_seconds and prompt_seconds

    def open(self, seed, prompt=None):
        """A new stream with selector key `seed`; returns its id.  It waits for frames.  prompt: None, or int mu-law codes [P], P >= 1
        (host or CUDA tensor), on fp16 pools only: the stream continues given audio, its first output being sample P.  It is scored
        in the step() after its frames cover samples [0, P), and generates from there."""
        if prompt is not None:
            prompt = check_prompt("prompt", prompt, None, None, self._eng.dtype == _lib.FP16, self._eng.A)
            if self._scorer is None:
                raise AssertionError("open: this pool has no scoring engine for prompts (NVWaveNet.open_live_pool makes one)")
            prompt = prompt.to(device=self.device, dtype=torch.int32)
        i = self._next_id
        self._next_id += 1
        self._streams[i] = _LiveStream(seed, self.channels, prompt)
        self._waiting.append(i)
        return i

    def _stream(self, i):
        if i not in self._streams:
            raise AssertionError(f"no open stream {i}")
        return self._streams[i]

    def push(self, i, frames):
        """Appends frames [C][n] (numpy array or torch tensor) to stream i.  Nothing is generated until step()."""
        s = self._stream(i)
        if s.finished:
            raise AssertionError(f"push: stream {i} is finished")
        shape = tuple(int(v) for v in frames.shape)
        if len(shape) != 2 or shape[0] != self.channels:
            raise AssertionError(f"push: frames must be [{self.channels}][n]; got {shape}")
        s.append(frames.detach().to("cpu", torch.float32).numpy() if isinstance(frames, torch.Tensor) else np.asarray(frames, np.float32))

    def finish(self, i):
        """Stream i gets no more frames: step() generates the rest of its samples and then closes it."""
        s = self._stream(i)
        s.finished = True
        if s.prompt is None and s.frames * self.stride == s.position or s.prompt is not None and s.frames * self.stride < s.prompt.numel():
            # nothing left to generate, or a prompt its frames never cover: its slot, if any, is free
            if i in self._waiting:
                self._waiting.remove(i)
            del self._streams[i]

    def state_seconds(self):
        """GPU seconds spent saving and loading slot states so far (timed pools; synchronises)."""
        torch.cuda.synchronize()
        return self._timer.seconds("save", "saved"), self._timer.seconds("load", "loaded")

    def prompt_seconds(self):
        """GPU seconds spent producing, scoring and saving prompts so far (timed pools; synchronises)."""
        torch.cuda.synchronize()
        return self._timer.seconds("prompt", "prompted")

    def _score_prompts(self):
        """Scores the waiting streams whose frames now cover their prompts, in groups of the scoring engine's rows
        (plan_prompt_groups); each becomes a parked stream at position P with the state its scoring row left."""
        st = self.stride
        ready = [(i, self._streams[i].prompt.numel()) for i in self._waiting
                 if self._streams[i].prompt is not None and self._streams[i].frames >= prompt_frames(self._streams[i].prompt.numel(), st)]
        if not ready:
            return
        if self._scorer_eng is None:
            self._scorer_eng = self._scorer()
            # on the device once, so a group's producer load copies no weights from the host
            self._network = tuple(torch.as_tensor(a).to(device=self.device, dtype=torch.float32).contiguous() for a in self._network)
        for group in plan_prompt_groups(ready, self._scorer_eng.B):
            self._timer.mark("prompt")
            states = self._score_group(group)
            self._timer.mark("prompted")
            for (i, P), state in zip(group, states):
                s = self._streams[i]
                s.state, s.position, s.started, s.prompt = state, P, True, None
                if s.finished and s.frames * st == P:                        # a prompt and nothing after it
                    self._waiting.remove(i)
                    del self._streams[i]

    def _score_group(self, group):
        """One scoring stream on the scoring engine: row j is group[j] = (id, P_j), rows by P.  Its conditioning comes from the
        rows' frames through the whole-batch producer; it is scored in pieces that end at each distinct P_j and at multiples of
        the window, rows past their prompt's end on code 128 (their results unused), and each row's state is saved where its prompt
        ends (nvwn_score_save_states, with the stream's seed).  Returns the states in group order."""
        eng = self._scorer_eng
        P_max = group[-1][1]
        F = prompt_frames(P_max, self.stride)
        feats = np.zeros((eng.B, self.channels, F), np.float32)
        for j, (i, _) in enumerate(group):
            s = self._streams[i]
            n = min(s.frames, F)
            feats[j, :, :n] = s.span(0, n)
        states = [None] * len(group)

        def fill(a, m):
            if a == 0:                          # the frames go in once, after the scorer has made its code rows
                eng.cond_producer_load(feats, *self._network, self.stride)
            eng.cond_producer_run_stream(a, m)

        def save(rows):
            for j, state in zip(rows, eng.score_save_states(rows, [self._streams[group[j][0]].seed for j in rows])):
                states[j] = state

        _score_prompt_group(eng, [self._streams[i].prompt for i, _ in group], fill, save)
        return states

    def step(self, audio=None, saturate=False):
        """One window at the engine's next sample: pushes each resident stream's pending frames (as many as its ring takes), scores the
        prompts whose frames are in (_score_prompts), parks the resident streams that are not ready and gives the free slots to ready waiting streams (plan_live_step), and if any slot is
        occupied generates `window` samples.  Returns {id: int32 CUDA tensor [k]} of the streams that advanced; with audio="float" or
        "int16" returns (samples, audio), audio {id: numpy [k]} decoded as LiveSession.push decodes.  A finished stream that has all
        its samples leaves the pool."""
        if audio not in (None, "float", "int16"):
            raise AssertionError(f"step: audio is None, 'float' or 'int16'; got {audio!r}")
        eng, K, st = self._eng, self.upsample_window, self.stride
        resident = {i: s for i, s in self._streams.items() if s.slot is not None}
        push = [(i, s, min(s.frames - s.pushed, live_push_limit(s.pushed, s.position, self.ring_frames, K, st))) for i, s in resident.items()]
        push = [(i, s, k) for i, s, k in push if k > 0]
        if push:
            eng.cond_producer_push_slots([s.slot for _, s, _ in push], [s.span(s.pushed, s.pushed + k) for _, s, k in push])
            for _, s, k in push:
                s.pushed += k
        self._score_prompts()
        park, place = plan_live_step({i: (s.slot, s.position, s.frames, s.finished) for i, s in resident.items()},
                                     [(i, self._streams[i].position, self._streams[i].frames, self._streams[i].finished) for i in self._waiting
                                      if self._streams[i].prompt is None],
                                     eng.B, self.window, st)
        if park:
            self._timer.mark("save")
            states = eng.save_slots([resident[i].slot for i in park])
            self._timer.mark("saved")
            for j, i in enumerate(park):
                s = resident.pop(i)
                s.state, s.slot = states[j], None
                self._waiting.append(i)
            self.parks += len(park)
        if place:
            placed = {i for i, _ in place}
            self._waiting = [i for i in self._waiting if i not in placed]
            new = [(i, b) for i, b in place if not self._streams[i].started]
            old = [(i, b) for i, b in place if self._streams[i].started]
            if new:
                eng.restart_slots([b for _, b in new], [self._streams[i].seed for i, _ in new])
            if old:
                states = torch.stack([self._streams[i].state for i, _ in old])         # before the span: it times the load alone
                self._timer.mark("load")
                eng.load_slots([b for _, b in old], states)
                self._timer.mark("loaded")
                self.resumes += len(old)
            spans = []
            for i, b in place:
                s = self._streams[i]
                first = live_frames(s.position, 1, K, st)[0]
                s.drop_before(first)
                s.pushed = min(s.frames, first + self.ring_frames)
                s.slot, s.state, s.started = b, None, True
                spans.append(s.span(first, s.pushed))
                resident[i] = s
            eng.cond_producer_attach_live([b for _, b in place], [self.t - self._streams[i].position for i, _ in place],
                                          [live_frames(self._streams[i].position, 1, K, st)[0] for i, _ in place], spans)
        out, auds = {}, {}
        if not resident:
            return out if audio is None else (out, auds)
        t, n = self.t, self.window
        eng.cond_producer_run_slots([s.slot for s in resident.values()], t, n)
        eng.set_selectors_random_slots(t, n)
        eng.run_stream(t, n, eng.B)
        self.launches += 1
        self.t += n
        pos = t % eng.N                                           # windows start at multiples of the window: no wrap inside
        if self._stage is None:
            self._stage = torch.empty((eng.B, eng.N), dtype=torch.int32, device=self.device)
        eng.get_yout(self._stage, pos, n)
        decoded = eng.get_audio(pos, n, int16=audio == "int16", saturate=saturate) if audio is not None else None
        for i, s in resident.items():
            k = min(n, s.frames * st - s.position)
            out[i] = self._stage[s.slot, pos:pos + k].clone()
            if decoded is not None:
                auds[i] = decoded[s.slot, :k].copy()
            s.position += k
            s.drop_before(live_frames(s.position, 1, K, st)[0])   # a resume reads from the first frame its next sample reads
            if s.finished and s.position == s.frames * st:        # all its samples delivered: the slot is free
                del self._streams[i]
        return out if audio is None else (out, auds)

    def close(self):
        for e in (self._eng, self._scorer_eng):
            if e is not None:
                e.close()
        self._eng = self._scorer_eng = None


class NVWaveNet:
    def __init__(self, embedding_prev, embedding_curr, conv_out_weight, conv_end_weight, dilate_weights, dilate_biases,
                 max_dilation, res_weights, res_biases, skip_weights, skip_biases, use_embed_tanh):
        self._lib = _lib.lib()
        R, S, A = self._lib.get_R(), self._lib.get_S(), self._lib.get_A()
        self.R, self.S, self.A = R, S, A
        self.max_dilation = max_dilation
        self.use_embed_tanh = use_embed_tanh

        # embeddings arrive [A][R] and are consumed as emb[a * R + r]: two transposes cancel, keep the values as they are
        _expect("embedding_prev", embedding_prev, (A, R))
        _expect("embedding_curr", embedding_curr, (A, R))
        self.embedding_prev = column_major(embedding_prev.t())
        self.embedding_curr = column_major(embedding_curr.t())
        _expect("conv_out_weight", conv_out_weight, (A, S))
        _expect("conv_end_weight", conv_end_weight, (A, A))
        self.conv_out = column_major(conv_out_weight)
        self.conv_end = column_major(conv_end_weight)

        n = len(dilate_weights)
        counts = {"dilate_biases": len(dilate_biases), "skip_weights": len(skip_weights), "skip_biases": len(skip_biases),
                  "res_weights": len(res_weights) + 1, "res_biases": len(res_biases) + 1}      # the last layer has no residual conv
        if any(c != n for c in counts.values()):
            raise AssertionError(f"Number of layers is inconsistent for different parameter types: dilate_weights {n}, {counts}")
        # the kernel still wants a residual matrix for the last layer: all zero (pytorch/nv_wavenet.py:139-141)
        like = dilate_weights[0] if n else embedding_prev
        res_weights = list(res_weights) + [torch.zeros(R, R, dtype=like.dtype, device=like.device)]
        res_biases = list(res_biases) + [torch.zeros(R, dtype=like.dtype, device=like.device)]

        self.layers = []                                 # per layer: (Wprev, Wcur, Bh, Wres, Bres, Wskip, Bskip), kernel layouts
        for l in range(n):
            w = dilate_weights[l]
            if w.size(2) != 2:
                raise AssertionError("nv-wavenet only supports kernel_size 2 dilated convolutions")
            _expect(f"dilate_weights[{l}]", w, (2 * R, R))
            _expect(f"dilate_biases[{l}]", dilate_biases[l], (2 * R,))
            _expect(f"res_weights[{l}]", res_weights[l], (R, R))
            _expect(f"res_biases[{l}]", res_biases[l], (R,))
            _expect(f"skip_weights[{l}]", skip_weights[l], (S, R))
            _expect(f"skip_biases[{l}]", skip_biases[l], (S,))
            self.layers.append((column_major(w[:, :, 0]), column_major(w[:, :, 1]), dilate_biases[l],
                                column_major(res_weights[l]), res_biases[l], column_major(skip_weights[l]), skip_biases[l]))
        self.num_layers = n
        self._engines = {}                               # (batch, samples, fp16) -> persistent NVWavenetInfer
        self.engines_created = 0

    def _engine(self, batch_size, sample_count, fp16):
        """The persistent engine for this problem size (created and loaded on first use)."""
        key = (batch_size, sample_count, bool(fp16))
        eng = self._engines.get(key)
        if eng is None:
            eng = self._new_engine(batch_size, sample_count, fp16)
            self._engines[key] = eng
            self.engines_created += 1
        return eng

    def _new_engine(self, batch_size, sample_count, fp16):
        """A new engine of this problem size with the model's weights."""
        from .infer import NVWavenetInfer
        eng = NVWavenetInfer(self.num_layers, self.max_dilation, batch_size, sample_count, 0, bool(self.use_embed_tanh),
                             R=self.R, S=self.S, A=self.A, dtype=_lib.FP16 if fp16 else _lib.FP32)
        f32 = lambda t: t.float().contiguous()
        eng.set_embeddings(f32(self.embedding_prev), f32(self.embedding_curr))
        for l, layer in enumerate(self.layers):
            eng.set_layer_weights(l, *[f32(t) for t in layer])
        zero = torch.zeros(self.A, dtype=torch.float32)                     # "We didn't use biases on our outputs" (wavenet_infer.cu:75-82)
        eng.set_out_weights(f32(self.conv_out), zero, f32(self.conv_end), zero)
        return eng

    def open_live(self, upsample_weight, upsample_bias, cond_weight, cond_bias, stride, batch_size, seed, window=4096, fp16=False, prompt=None):
        """Live vocoding: a LiveSession that generates `batch_size` utterances while their mel frames [batch][C][n] are still
        arriving (LiveSession.push).  The conditioning network is that of set_conditioning_from_features (upsample_weight [C][C][w],
        upsample_bias [C], cond_weight [L*2R][C] or [L*2R][C][1], cond_bias [L*2R]; numpy arrays or torch tensors); the frames go
        into a ring on the device of live_ring_frames(window, w, stride) frames per utterance.  Selectors are Philox under `seed`,
        drawn by absolute sample, so the pushes together give infer(cond, seed=seed, fp16=fp16, window=window) of the finished
        frames' conditioning (nvwn_cond_from_features_host), bit for bit.  The session has an engine of its own, apart from the
        engines infer() and the other calls share.
        prompt: None, or int mu-law codes [batch_size][P], P >= 1 (host or CUDA tensor), fp16 only: the utterances continue given
        audio.  The pushes then give infer(cond, seed=seed, fp16=True, window=window, prompt=prompt)[:, P:], bit for bit: the
        frames' first P samples are scored as they arrive, and generation starts at sample P once they all are."""
        Cc, up, network = self._cond_network("open_live", upsample_weight, upsample_bias, cond_weight, cond_bias, stride)
        _check_rows("open_live", "batch_size", batch_size, window)
        if prompt is not None:
            prompt = self._check_prompt("prompt", prompt, batch_size, None, fp16).to(device="cuda", dtype=torch.int32)
        eng = self._new_engine(batch_size, window, fp16)
        eng.cond_producer_open_live(*network, stride, live_ring_frames(window, up, stride))
        return LiveSession(eng, Cc, up, stride, seed, window, prompt)

    def open_live_pool(self, upsample_weight, upsample_bias, cond_weight, cond_bias, stride, slots, window, fp16=False, timed=False):
        """Live serving: a LivePool whose streams, each with its own mel frames [C][n] arriving at its own pace, share one engine of
        `slots` rows and `window` samples; `window` is also the samples per launch, so it trades latency against launches.  The
        conditioning network is that of set_conditioning_from_features (upsample_weight [C][C][w], upsample_bias [C], cond_weight
        [L*2R][C] or [L*2R][C][1], cond_bias [L*2R]; numpy arrays or torch tensors).  Each stream's outputs, concatenated, equal
        infer(cond, seed=seed, fp16=fp16) of its finished frames' conditioning (nvwn_cond_from_features_host), bit for bit.  The
        pool has an engine of its own, apart from the engines infer() and the other calls share.  timed: see LivePool.
        On fp16 pools LivePool.open takes a prompt; the pool then makes, on the first prompt, a scoring engine of `slots` rows and
        `window` samples with the same weights."""
        Cc, up, network = self._cond_network("open_live_pool", upsample_weight, upsample_bias, cond_weight, cond_bias, stride)
        _check_rows("open_live_pool", "slots", slots, window)
        eng = self._new_engine(slots, window, fp16)
        eng.cond_producer_set_weights(*network, stride)
        scorer = (lambda: self._new_engine(slots, window, True)) if fp16 else None
        return LivePool(eng, Cc, up, stride, timed, scorer, network)

    def _cond_network(self, what, upsample_weight, upsample_bias, cond_weight, cond_bias, stride):
        """(C, window, network) of a conditioning network checked for this model (check_cond_network, its errors naming `what`),
        network being (upsample_weight, upsample_bias, cond_weight [L*2R][C], cond_bias) as the producer calls take them."""
        Cc, up = check_cond_network(self.num_layers, self.R, upsample_weight, upsample_bias, cond_weight, cond_bias, stride, AssertionError,
                                    what)
        return Cc, up, (upsample_weight, upsample_bias, cond_weight.reshape(self.num_layers * 2 * self.R, Cc), cond_bias)

    def _check_utterances(self, cond_inputs):
        """The sample counts n_u of per-utterance conditioning [2R][L][n_u] (channels x num_layers x samples)."""
        for c in cond_inputs:
            if c.dim() != 3 or (c.size(0), c.size(1)) != (2 * self.R, self.num_layers):
                raise AssertionError(f"each input is channels x num_layers x samples; got {tuple(c.size())}")
        return [int(c.size(2)) for c in cond_inputs]

    def _gather(self, cond_inputs, count, rows, pieces):
        """A store slab [count][L][rows][2R] of per-utterance conditioning [2R][L][n_u]: piece (row, u, a, o, m) puts samples
        [a, a + m) of utterance u at positions [o, o + m) of its row; everything else is zero."""
        lh = torch.zeros((count, self.num_layers, rows, 2 * self.R), dtype=torch.float32, device="cuda")
        for j, u, a, o, m in pieces:
            lh[o:o + m, :, j].copy_(cond_inputs[u][:, :, a:a + m].permute(2, 1, 0))
        return lh

    def _cond_size(self, cond_input):
        """(batch, samples) of conditioning channels x batch x num_layers x samples."""
        if cond_input.dim() != 4 or (cond_input.size(0), cond_input.size(2)) != (2 * self.R, self.num_layers):
            raise AssertionError(f"Inputs are channels x batch x num_layers x samples; got {tuple(cond_input.size())}")
        return cond_input.size(1), cond_input.size(3)

    def _check_prompt(self, what, prompt, rows, n, fp16):
        return check_prompt(what, prompt, rows, n, fp16, self.A)

    def infer(self, cond_input, implementation, seed=None, fp16=False, window=None, prompt=None):
        """cond_input: channels x batch x num_layers x samples (pytorch/nv_wavenet.py:172-196); returns int32 [batch][samples].
        `implementation` (Impl.*) is accepted for compatibility: one kernel family serves all of them.
        Generation runs in windows of W samples (nvwn_run_stream) through one engine of W samples per (batch, W, precision):
        W = samples without a window, so one window of the whole length; with window=W any length fits, and the result is the
        same as without a window, bit for bit.
        prompt: int mu-law codes [batch][P], 1 <= P < samples, each in [0, A) (host or CUDA tensor), fp16 only.  The prompt is
        scored all steps at once, a window at a time (nvwn_score_stream), generation is primed from the scoring state
        (nvwn_prime_from_score) and continues with samples [P, samples), drawn with the selectors infer() uses at those samples.
        The first P columns of the result are the prompt.  The continuation is not bit-identical to forced generation of the
        prompt (the history holds the scorer's fp16 values, DESIGN.md §5.4); with a window it is bit-identical to without one."""
        batch_size, sample_count = self._cond_size(cond_input)
        _check_window(window)
        if prompt is not None:
            prompt = self._check_prompt("prompt", prompt, batch_size, sample_count, fp16).to(device="cuda", dtype=torch.int32)
        eng = self._engine(batch_size, window or sample_count, fp16)
        lh = column_major(cond_input).float()                       # [samples][layers][batch][2R]
        eng.reset_history()
        sel = None
        if seed is None:                                            # the reference's host draw, on the caller's rand() stream
            sel = np.empty(sample_count * batch_size, np.float32)
            _lib.check(self._lib.nvwn_libc_selectors(C.c_void_p(sel.ctypes.data), batch_size, sample_count), "selectors")
        samples = torch.empty((batch_size, sample_count), dtype=torch.int32, device="cuda")
        self._generate(eng, lh, prompt, seed, sel, samples)
        torch.cuda.synchronize()
        return samples

    @staticmethod
    def _generate(eng, lh, prompt, seed, sel, samples):
        """The window loop of infer() on a reset engine of W samples: windows at multiples of W, each one's conditioning set once.
        With a prompt [batch][P], the prompt's part of a window is scored, the engine primed at the prompt's end and the rest of the
        window generated; without one (P = 0) every window is generated whole.  Selectors of the generated samples: Philox under
        `seed`, or the host draw `sel` placed at their positions."""
        batch_size, sample_count = samples.shape
        window = eng.N
        if prompt is not None:
            samples[:, :prompt.shape[1]] = prompt

        def select(g0, k):
            if sel is None:
                eng.set_selectors_random_stream(seed, g0, k)
            else:
                chunk, o = np.zeros(window * batch_size, np.float32), g0 % window
                chunk[o * batch_size:(o + k) * batch_size] = sel[g0 * batch_size:(g0 + k) * batch_size]
                eng.set_selectors(chunk)

        for first in range(0, sample_count, window):
            n = min(window, sample_count - first)
            eng.set_conditioning(lh[first:first + n], 0, n)
            _score_then_generate(eng, prompt, first, n, select, lambda g0, k: eng.get_yout_stream(samples[:, g0:g0 + k], g0, k))

    def infer_many(self, cond_inputs, seeds, slots=64, window=4096, fp16=False, timing=None, prompts=None):
        """Continuous batching: generates a queue of utterances of different lengths through one engine of `slots` utterances and
        `window` samples.  cond_inputs: per utterance, conditioning [2R][L][n_u] (channels x num_layers x samples); seeds: one
        integer per utterance (device selectors, as infer(seed=...)).  Returns int32 CUDA tensors [n_u], each bit-identical to
        infer() of that utterance alone with its seed.  The engine runs in windows of `window` samples; at each window boundary
        the slots whose utterance has ended take the next queued ones in arrival order (plan_slots).  A slot with nothing to do
        keeps running on stale inputs and its output is discarded.
        prompts: None, or per utterance None or int mu-law codes [P_u], 1 <= P_u < n_u (host or CUDA tensor), fp16 only; cond_inputs
        still cover the whole utterance.  A prompted utterance generates n_u - P_u samples (the schedule is plan_slots of those),
        and is bit-identical to infer(cond_u, seed=s_u, fp16=True, prompt=p_u) of it alone: at the boundary where it starts, the
        prompted utterances starting there are scored together through the engine's own conditioning store (nvwn_score_stream) and
        each slot is primed from its row once its prompt has been scored (nvwn_prime_slots_from_score).  The first P_u outputs
        are the prompt.  timing: a dict, or None; if given, receives the GPU seconds spent in restarts and per-slot uploads
        ("restart_upload_s"), in generation ("generate_s") and in scoring and priming prompts ("prime_s")."""
        if len(cond_inputs) != len(seeds):
            raise AssertionError(f"{len(cond_inputs)} utterances but {len(seeds)} seeds")
        lengths = self._check_utterances(cond_inputs)
        prompts = self._slot_prompts(prompts, lengths, fp16)
        skip = [0 if p is None else int(p.numel()) for p in prompts]                  # samples before the generated ones
        plan = plan_slots([n - P for n, P in zip(lengths, skip)], slots, window)
        windows = _windows(plan, [n - P for n, P in zip(lengths, skip)], window)
        eng = self._engine(slots, window, fp16)
        st = torch.cuda.current_stream()
        timer = _Timer(timing)
        prime = lambda k: self._prime(eng, windows[k], plan, prompts, skip, cond_inputs, seeds, timer)
        outs = self._serve_queue(eng, plan, windows, lengths, skip, cond_inputs, seeds, timer, prime, prompts)
        timer.report(prime_s=("prime", "primed"))
        return outs

    def _prime(self, eng, window, plan, prompts, skip, cond_inputs, seeds, timer, score_models=None):
        """The prompts of a prompted queue that start at one window boundary (window: its _windows entry): the prompted utterances
        starting there, by prompt length, are the rows of one scoring stream through the engine's own conditioning store (free now
        that the last window was generated), and each slot is primed from its row.  score_models: None, or called with those
        utterances before they are scored.  timer: marked "prime" before and "primed" after, when there are any."""
        st = torch.cuda.current_stream()
        group = sorted((u for u in window[2] if prompts[u] is not None), key=lambda u: skip[u])
        if not group:
            return
        timer.mark("prime")
        if score_models is not None:
            score_models(group)

        def fill(a, m):
            lh = self._gather(cond_inputs, m, len(group), [(j, u, a, 0, min(skip[u], a + m) - a) for j, u in enumerate(group) if skip[u] > a])
            eng.set_conditioning_slots(lh, list(range(len(group))), a, stream=st)

        def at_end(rows):
            eng.prime_slots_from_score(rows, [plan[group[j]][0] for j in rows], [seeds[group[j]] for j in rows], stream=st)

        _score_prompt_group(eng, [prompts[u] for u in group], fill, at_end, stream=st)
        timer.mark("primed")

    def _serve_queue(self, eng, plan, windows, lengths, skip, cond_inputs, seeds, timer, before, prompts=None):
        """The queue of infer_many and ModelSet.infer_many once it is planned: the engine reset, then _serve with before(k) and
        each window's conditioning of its live slots gathered from cond_inputs (utterance u's generated samples reading it from
        sample skip[u] on).  timer: a _Timer that receives the GPU seconds of restarts and per-slot uploads ("restart_upload_s")
        and of generation ("generate_s")."""
        _reset(eng)
        st = torch.cuda.current_stream()

        def condition(k):
            first, count, _, live = windows[k]
            if live:
                lh = self._gather(cond_inputs, count, len(live), [(j, u, skip[u] + a, 0, m) for j, (_, u, a, m) in enumerate(live)])
                eng.set_conditioning_slots(lh, [s for s, _, _, _ in live], first, stream=st)

        outs = self._serve(eng, plan, windows, lengths, skip, seeds, timer, condition, before=before, prompts=prompts)
        timer.report(restart_upload_s=("condition", "launch"), generate_s=("launch", "done"))
        return outs

    def _slot_prompts(self, prompts, lengths, fp16):
        """infer_many's prompts checked: per utterance None or int32 CUDA codes [P_u], 1 <= P_u < n_u, each in [0, A), and fp16 if any
        is given.  Returns the list (all None without prompts)."""
        if prompts is None:
            return [None] * len(lengths)
        if len(prompts) != len(lengths):
            raise AssertionError(f"{len(lengths)} utterances but {len(prompts)} prompts")
        out = [None if p is None else self._check_prompt(f"prompt {u}", p, None, lengths[u], fp16) for u, p in enumerate(prompts)]
        return [None if p is None else p.to(device="cuda", dtype=torch.int32) for p in out]

    def infer_many_from_features(self, features, seeds, upsample_weight, upsample_bias, cond_weight, cond_bias, stride, slots=64,
                                 window=4096, fp16=False, timing=None):
        """Continuous batching from mel frames: infer_many with each utterance given as its frames [C][T_u] instead of expanded
        conditioning.  Utterance u has T_u * stride samples.  The weights are those of set_conditioning_from_features
        (upsample_weight [C][C][w], upsample_bias [C], cond_weight [L*2R][C] or [L*2R][C][1], cond_bias [L*2R]).  Returns int32
        CUDA tensors [T_u * stride], each bit-identical to infer() of that utterance alone with its seed and the conditioning the
        producer's arithmetic gives it (nvwn_cond_from_features_host).
        The schedule is infer_many's, through an engine of two windows: on a side stream the per-slot conditioning producer makes
        window k + 1 of the slots live then, while the current stream generates window k.  frames and weights may be numpy arrays
        or torch tensors (CUDA ones are read in stream order).  timing: a dict, or None; if given, receives the GPU seconds of
        production on the side stream ("produce_s"), the time generation waited for it ("produce_wait_s"), of restarts and
        selectors ("restart_select_s") and of generation ("generate_s")."""
        if len(features) != len(seeds):
            raise AssertionError(f"{len(features)} utterances but {len(seeds)} seeds")
        Cc, _, network = self._cond_network("infer_many_from_features", upsample_weight, upsample_bias, cond_weight, cond_bias, stride)
        lengths = [T * stride for T in _check_frames(features, Cc)]
        # contiguous fp32 frames, made on the current stream before the side stream is ordered after it
        features = [f.to(torch.float32).contiguous() if isinstance(f, torch.Tensor) else np.ascontiguousarray(f, np.float32) for f in features]
        plan = plan_slots(lengths, slots, window)
        windows = _windows(plan, lengths, window)
        eng = self._engine(slots, 2 * window, fp16)
        _reset(eng)
        eng.cond_producer_set_weights(*network, stride)

        cur, side = torch.cuda.current_stream(), torch.cuda.Stream()
        side.wait_stream(cur)                                         # frames made on the current stream
        timer = _Timer(timing)
        ready, read, keep = {}, {}, []

        def produce(k):
            # window k on the side stream, into the positions of window k - 2: after that window has been generated and read
            if k >= len(windows):
                return
            first, count, starting, live = windows[k]
            if k - 2 in read:
                side.wait_event(read.pop(k - 2))
            timer.mark("produce", side)
            if starting:
                keep.append(eng.cond_producer_set_slots([plan[u][0] for u in starting], [features[u] for u in starting],
                                                        [first] * len(starting), stream=side))
            if live:
                eng.cond_producer_run_slots([s for s, _, _, _ in live], first, count, stream=side)
            timer.mark("produced", side)
            ready[k] = torch.cuda.Event()
            ready[k].record(side)

        def condition(k):
            cur.wait_event(ready.pop(k))

        def after(k):
            read[k] = torch.cuda.Event()
            read[k].record(cur)
            produce(k + 1)                                            # enqueued after window k's generation, which it overlaps

        produce(0)
        outs = self._serve(eng, plan, windows, lengths, [0] * len(lengths), seeds, timer, condition, after)
        timer.report(produce_s=("produce", "produced"), produce_wait_s=("condition", "restart"), restart_select_s=("restart", "launch"),
                     generate_s=("launch", "done"))
        return outs

    def _serve(self, eng, plan, windows, lengths, skip, seeds, timer, condition, after=None, before=None, prompts=None):
        """The window loop of infer_many and infer_many_from_features on the current stream.  Per window k: before(k), which
        primes the prompted slots that start there; condition(k), which leaves the conditioning of the window's live slots in the
        engine or makes the stream wait for it; the restarts of the other slots whose utterance starts there; their selectors;
        the launch; the outputs; then after(k); a synchronise at the end.  skip: per utterance the length P_u of its prompt, 0 for
        none; prompts: None, or per utterance its prompt [P_u] (CUDA) or None: the output's first P_u samples, generated ones after
        them (windows count generated samples; outputs have `lengths`).  Returns the outputs; `timer` (a _Timer) is marked per window before condition ("condition"), the restarts ("restart"), the
        launch ("launch") and after the outputs ("done")."""
        outs = [torch.empty(n, dtype=torch.int32, device="cuda") for n in lengths]
        for o, p in zip(outs, prompts or ()):
            if p is not None:
                o[:p.numel()].copy_(p)
        stage = torch.empty((eng.B, eng.N), dtype=torch.int32, device="cuda")
        st = torch.cuda.current_stream()
        for k, (first, count, starting, live) in enumerate(windows):
            if before is not None:
                before(k)
            timer.mark("condition")
            condition(k)
            timer.mark("restart")
            restart = [u for u in starting if not skip[u]]
            if restart:
                eng.restart_slots([plan[u][0] for u in restart], [seeds[u] for u in restart], stream=st)
            eng.set_selectors_random_slots(first, count, stream=st)
            timer.mark("launch")
            eng.run_stream(first, count, eng.B, stream=st)
            pos = first % eng.N                                       # windows start at multiples of the window: no wrap inside
            eng.get_yout(stage, pos, count, stream=st)
            for s, u, a, m in live:
                outs[u][skip[u] + a:skip[u] + a + m].copy_(stage[s, pos:pos + m])
            timer.mark("done")
            if after is not None:
                after(k)
        torch.cuda.synchronize()
        return outs

    def log_likelihood(self, cond_input, audio, window=None):
        """Per-sample log-likelihood of `audio` (int mu-law codes [batch][samples]) given `cond_input` (channels x batch x
        num_layers x samples, as for infer()): log p(audio[b][t] | audio[b][0..t), conditioning) under the fp16 model, all steps
        of a window at once.  Returns a float32 CUDA tensor [batch][samples].
        Scoring runs in windows of W samples (nvwn_score_stream) through one fp16 engine of W samples per (batch, W): W = samples
        without a window, so one window of the whole length; with window=W the engine holds W samples of conditioning instead of
        all of them, and the result is the same as without a window, bit for bit.  Either way the engine's scoring stream is left
        open, so the last window also carries every layer's front for a call that would continue it."""
        batch_size, sample_count = self._check_scoring(cond_input, audio, window)
        return self._score_cond(self._engine(batch_size, window or sample_count, True), cond_input, audio)

    def _check_scoring(self, cond_input, audio, window):
        """(batch, samples) of log_likelihood's arguments, checked"""
        batch_size, sample_count = self._cond_size(cond_input)
        if tuple(audio.size()) != (batch_size, sample_count):
            raise AssertionError(f"audio must be [batch][samples] = {(batch_size, sample_count)}; got {tuple(audio.size())}")
        _check_window(window)
        return batch_size, sample_count

    def _score_cond(self, eng, cond_input, audio):
        """log_likelihood on the fp16 engine `eng`, its arguments checked"""
        # converted a window at a time, so a windowed call never holds an fp32 copy of the whole length
        fill = lambda first, n: eng.set_conditioning(column_major(cond_input[..., first:first + n]).float(), 0, n)
        return self._score(eng, audio.to(device="cuda", dtype=torch.int32), fill)

    def log_likelihood_from_features(self, features, audio, upsample_weight, upsample_bias, cond_weight, cond_bias, stride, window=None,
                                     timing=None):
        """log_likelihood with the conditioning made on the device from mel frames: features [batch][C][T], audio int mu-law codes
        [batch][T * stride], and the conditioning network of set_conditioning_from_features (upsample_weight [C][C][w],
        upsample_bias [C], cond_weight [L*2R][C] or [L*2R][C][1], cond_bias [L*2R]); numpy arrays or torch tensors.  Returns a
        float32 CUDA tensor [batch][T * stride], equal bit for bit to log_likelihood of the conditioning the producer's arithmetic
        gives (nvwn_cond_from_features_host).
        The frames are loaded into the engine once (nvwn_cond_producer_load); each window's conditioning is then produced from
        them just before it is scored (nvwn_cond_producer_run_stream).  window=None uses one engine of the whole length; window=W
        one engine of W samples, so neither the expanded conditioning nor a store of the whole length ever exists.  timing: a dict,
        or None; if given, receives the GPU seconds of production over the windows ("produce_s", the load not included) and of
        scoring ("score_s")."""
        shp = lambda a: tuple(int(v) for v in a.shape)
        Cc, _, network = self._cond_network("log_likelihood_from_features", upsample_weight, upsample_bias, cond_weight, cond_bias, stride)
        if len(shp(features)) != 3 or shp(features)[1] != Cc or shp(features)[2] < 1:
            raise AssertionError(f"features must be [batch][{Cc}][T] with T >= 1; got {shp(features)}")
        batch_size, sample_count = shp(features)[0], shp(features)[2] * stride
        if shp(audio) != (batch_size, sample_count):
            raise AssertionError(f"audio must be [batch][T * stride] = {(batch_size, sample_count)}; got {shp(audio)}")
        _check_window(window)
        audio = torch.as_tensor(audio).to(device="cuda", dtype=torch.int32)
        eng = self._engine(batch_size, window or sample_count, True)
        eng.cond_producer_load(features, *network, stride)
        return self._score(eng, audio, eng.cond_producer_run_stream, timing)

    def _check_queue(self, what, lengths, audios, slots, window):
        """The audios of a scoring queue as int32 CUDA codes [n_u], checked against `lengths` (each >= 1), and slots and window
        checked, before any engine exists."""
        if len(audios) != len(lengths):
            raise AssertionError(f"{what}: {len(lengths)} utterances but {len(audios)} audios")
        if any(n < 1 for n in lengths):
            raise AssertionError(f"{what}: every utterance needs at least one sample")
        for u, (a, n) in enumerate(zip(audios, lengths)):
            if tuple(a.shape) != (n,):
                raise AssertionError(f"{what}: audio {u} must be [{n}] codes; got {tuple(a.shape)}")
        _check_rows(what, "slots", slots, window)
        return [torch.as_tensor(a).to(device="cuda", dtype=torch.int32) for a in audios]

    def log_likelihood_many(self, cond_inputs, audios, slots=64, window=4096, timing=None):
        """Packed scoring of a queue: log_likelihood of utterances of different lengths through one fp16 engine of `slots` rows and
        `window` samples, with no padding between utterances.  cond_inputs: per utterance, conditioning [2R][L][n_u] (channels x
        num_layers x samples); audios: per utterance, int mu-law codes [n_u] (host or CUDA).  Returns float32 CUDA tensors [n_u],
        each bit-identical to log_likelihood(c_u[:, None], a_u[None])[0] of that utterance alone.  Each utterance goes to the row
        that frees first (plan_packed) and starts there at the very next sample; the rows are scored in windows at multiples of
        `window` (nvwn_score_stream_packed), each window's conditioning set once, zero where a row has nothing.  timing: a dict, or
        None; if given, receives the GPU seconds of filling the conditioning ("produce_s") and of scoring ("score_s")."""
        lengths = self._check_utterances(cond_inputs)
        audios = self._check_queue("log_likelihood_many", lengths, audios, slots, window)
        plan = plan_packed(lengths, slots)
        eng = self._engine(slots, window, True)

        def fill(first, count, segs):
            eng.set_conditioning(self._gather(cond_inputs, count, slots, segs), 0, count)

        return self._score_packed(eng, plan, lengths, audios, fill, timing)

    def log_likelihood_many_from_features(self, features, audios, upsample_weight, upsample_bias, cond_weight, cond_bias, stride, slots=64,
                                          window=4096, timing=None):
        """log_likelihood_many with each utterance given as its mel frames [C][T_u] instead of expanded conditioning; utterance u has
        T_u * stride samples and audios[u] is [T_u * stride] codes.  The conditioning network is that of set_conditioning_from_features
        (upsample_weight [C][C][w], upsample_bias [C], cond_weight [L*2R][C] or [L*2R][C][1], cond_bias [L*2R]).  Returns float32
        CUDA tensors, each bit-identical to log_likelihood of that utterance alone on the conditioning the producer's arithmetic gives
        it (nvwn_cond_from_features_host).  Each window's conditioning comes from the per-slot producer: an utterance's frames are
        attached to its row at its start, and the producer runs once per distinct segment range of the window, in time order.
        timing as for log_likelihood_many."""
        Cc, _, network = self._cond_network("log_likelihood_many_from_features", upsample_weight, upsample_bias, cond_weight, cond_bias,
                                            stride)
        lengths = [T * stride for T in _check_frames(features, Cc)]
        audios = self._check_queue("log_likelihood_many_from_features", lengths, audios, slots, window)
        plan = plan_packed(lengths, slots)
        eng = self._engine(slots, window, True)
        eng.cond_producer_set_weights(*network, stride)
        keep = []

        def fill(first, count, segs):
            ranges = {}
            for s, u, a, o, m in segs:
                ranges.setdefault((o, m), []).append((s, u, a))
            # by first sample: a row's earlier segment is produced before the row's next utterance is attached
            for (o, m), group in sorted(ranges.items()):
                new = [(s, u) for s, u, a in group if a == 0]
                if new:
                    keep.append(eng.cond_producer_set_slots([s for s, _ in new], [features[u] for _, u in new], [plan[u][1] for _, u in new]))
                eng.cond_producer_run_slots([s for s, _, _ in group], first + o, m)

        return self._score_packed(eng, plan, lengths, audios, fill, timing)

    @staticmethod
    def _score_packed(eng, plan, lengths, audios, fill, timing):
        """The window loop of log_likelihood_many and log_likelihood_many_from_features: the plan_packed schedule `plan` of `lengths`
        over the fp16 engine `eng` of as many rows and W samples, in windows at multiples of W.  Per window: fill(first, count, segments)
        puts the conditioning of the window's segments into the store, then the window's audio and start flags are scored
        (nvwn_score_stream_packed) and each segment's logp copied out.  timing as for _score."""
        outs = [torch.empty(n, dtype=torch.float32, device="cuda") for n in lengths]

        def score(first, count, segs):
            audio, starts = _pack_window(count, segs, audios, eng.B)
            logp = eng.score_stream_packed(audio, starts, first)
            for s, u, a, o, m in segs:
                outs[u][a:a + m].copy_(logp[s, o:o + m])

        _score_windows(_packed_windows(plan, lengths, eng.N), fill, score, timing)
        return outs

    @staticmethod
    def _score(eng, audio, fill, timing=None):
        """The window loop of log_likelihood and log_likelihood_from_features: audio int32 CUDA [batch][samples] scored through the
        fp16 engine `eng` of W samples in windows at multiples of W, each after fill(first, n) has put the conditioning of samples
        [first, first + n) into the store.  timing: None, or a dict for the GPU seconds of fill ("produce_s") and of scoring
        ("score_s")."""
        batch_size, sample_count = audio.shape
        logp = torch.empty((batch_size, sample_count), dtype=torch.float32, device="cuda")
        _score_windows([(first, min(eng.N, sample_count - first)) for first in range(0, sample_count, eng.N)], fill,
                       lambda first, n: logp[:, first:first + n].copy_(eng.score_stream(audio[:, first:first + n], first)), timing)
        return logp


def group_models(plan, lengths, models, first, count, group, slots):
    """The model of each of the ceil(slots / group) slot groups in the window [first, first + count) of a plan_slots schedule
    with `models`: that of the group's utterances live in the window, 0 for a group with none."""
    table = [0] * ((slots + group - 1) // group)
    for u, (s, start) in enumerate(plan):
        if start < first + count and start + lengths[u] > first:
            table[s // group] = models[u]
    return table


class ModelSet:
    """Multi-model serving: several NVWaveNets of one shape (one voice each, say) served by one engine, each group of its slots
    generating with the weights of the utterance it holds (nvwn_set_model, DESIGN.md §6).  The set owns its engines, one per
    (slots, window, precision), each holding every net as a model (net m is model m); close() frees them."""

    def __init__(self, nets):
        nets = list(nets)
        if not nets:
            raise AssertionError("ModelSet needs at least one NVWaveNet")
        shape = lambda n: (n.R, n.S, n.A, n.num_layers, n.max_dilation, bool(n.use_embed_tanh))
        if any(shape(n) != shape(nets[0]) for n in nets):
            raise AssertionError(f"the nets of a ModelSet share R, S, A, layers, max_dilation and use_embed_tanh; got {[shape(n) for n in nets]}")
        from .infer import MAX_MODELS
        if len(nets) > MAX_MODELS:
            raise AssertionError(f"a ModelSet holds at most {MAX_MODELS} nets; got {len(nets)}")
        self.nets = nets
        self._engines = {}

    def _engine(self, slots, window, fp16):
        """The engine of (slots, window, precision), holding net m as model m (made on first use)."""
        key = (slots, window, bool(fp16))
        eng = self._engines.get(key)
        if eng is None:
            eng = self.nets[0]._new_engine(slots, window, fp16)
            for m, net in enumerate(self.nets[1:], 1):
                donor = net._new_engine(1, 1, fp16)
                try:
                    eng.set_model(m, donor)
                finally:
                    donor.close()
            self._engines[key] = eng
        return eng

    def _check_models(self, models, n, what="utterances"):
        """models as ints, checked: one per utterance (or row), each in [0, len(nets))"""
        if len(models) != n:
            raise AssertionError(f"{len(models)} models for {n} {what}")
        if any(int(m) != m or not 0 <= m < len(self.nets) for m in models):
            raise AssertionError(f"every model index is in [0, {len(self.nets)})")
        return [int(m) for m in models]

    def infer_many(self, models, cond_inputs, seeds, slots=64, window=4096, fp16=False, timing=None, prompts=None):
        """NVWaveNet.infer_many over several models: utterance u runs net models[u].  One engine of `slots` slots and `window`
        samples serves the whole queue; its slots are in groups of eng.model_group that run one model at a time, scheduled by
        plan_slots(..., models, group), and before each window's restarts the engine's group table is set to the models of the
        window's live utterances.  Returns int32 CUDA tensors [n_u], each bit-identical to
        nets[models[u]].infer(cond_u[:, None], Impl.AUTO, seed=seeds[u], fp16=fp16)[0].
        prompts: None, or per utterance None or int mu-law codes [P_u], as NVWaveNet.infer_many takes them (fp16 only).  At a
        boundary where prompted utterances start, the group table is set first, then the scoring table gives each of their
        scoring rows its utterance's model (nvwn_set_score_models), and they are scored and primed as NVWaveNet.infer_many does;
        each is bit-identical to nets[models[u]].infer(cond_u[:, None], Impl.AUTO, seed=seeds[u], fp16=True, prompt=p_u)[0].
        timing: a dict, or None; if given, receives the GPU seconds spent in restarts and per-slot uploads ("restart_upload_s"), in
        generation ("generate_s") and, with prompts, in scoring and priming them ("prime_s")."""
        net = self.nets[0]
        if not (len(models) == len(cond_inputs) == len(seeds)):
            raise AssertionError(f"{len(models)} models, {len(cond_inputs)} utterances and {len(seeds)} seeds")
        models = self._check_models(models, len(cond_inputs))
        lengths = net._check_utterances(cond_inputs)
        prompts = net._slot_prompts(prompts, lengths, fp16)
        skip = [0 if p is None else int(p.numel()) for p in prompts]
        made = [n - P for n, P in zip(lengths, skip)]                      # the generated samples
        eng = self._engine(slots, window, fp16)
        group = eng.model_group
        plan = plan_slots(made, slots, window, models, group)
        windows = _windows(plan, made, window)
        st = torch.cuda.current_stream()
        timer = _Timer(timing)

        def before(k):
            first, count, _, _ = windows[k]
            eng.set_group_models(group_models(plan, made, models, first, count, group, slots), stream=st)
            net._prime(eng, windows[k], plan, prompts, skip, cond_inputs, seeds, timer,
                       lambda us: eng.set_score_models([models[u] for u in us] + [0] * (slots - len(us)), stream=st))

        outs = net._serve_queue(eng, plan, windows, lengths, skip, cond_inputs, seeds, timer, before, prompts)
        if any(p is not None for p in prompts):
            timer.report(prime_s=("prime", "primed"))
        return outs

    def log_likelihood(self, models, cond_input, audio, window=None):
        """NVWaveNet.log_likelihood over several models: batch row b is scored with net models[b] (nvwn_set_score_models), all rows
        in one fp16 engine of the batch and W samples.  Returns a float32 CUDA tensor [batch][samples] whose row b is, bit for bit,
        nets[models[b]].log_likelihood of that row, windowed or not."""
        net = self.nets[0]
        batch_size, sample_count = net._check_scoring(cond_input, audio, window)
        models = self._check_models(models, batch_size, "batch rows")
        eng = self._engine(batch_size, window or sample_count, True)
        eng.set_score_models(models)
        return net._score_cond(eng, cond_input, audio)

    def log_likelihood_many(self, models, cond_inputs, audios, slots=64, window=4096, timing=None):
        """NVWaveNet.log_likelihood_many over several models: utterance u is scored with net models[u].  The rows of one fp16 engine
        of `slots` rows and `window` samples are split among the queue's models (plan_packed_models), each row keeping its model for
        the whole stream, and packed within each model as plan_packed does.  Returns float32 CUDA tensors [n_u], each bit-identical
        to nets[models[u]].log_likelihood_many([c_u], [a_u])[0].  timing as for NVWaveNet.log_likelihood_many."""
        net = self.nets[0]
        lengths = net._check_utterances(cond_inputs)
        models = self._check_models(models, len(lengths))
        _check_rows("log_likelihood_many", "slots", slots, window)
        plan, table = plan_packed_models(lengths, models, slots)
        audios = net._check_queue("log_likelihood_many", lengths, audios, slots, window)
        eng = self._engine(slots, window, True)
        eng.set_score_models(table)

        def fill(first, count, segs):
            eng.set_conditioning(net._gather(cond_inputs, count, slots, segs), 0, count)

        return net._score_packed(eng, plan, lengths, audios, fill, timing)

    def close(self):
        for eng in self._engines.values():
            eng.close()
        self._engines = {}
