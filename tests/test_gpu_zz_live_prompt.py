"""Prompted live streams: a LivePool stream opened with a prompt is scored once its frames cover the prompt, waits as a parked stream
at position P and is resumed like one; open_live(prompt=) scores the prompt as its frames arrive.  Each equals infer(prompt=) of its
finished frames' conditioning from sample P on, bit for bit, on every fp16 engine kind; and a state the scorer saved resumes in a
second engine of another batch and window."""
import numpy as np
import pytest

from tests import refgen
from tests.test_gpu_zz_cond_slots import CC, STRIDE, _host, _network
from tests.test_gpu_zz_park import _Run, _make
from tests.test_gpu_zz_selectors import _net
from tests.test_gpu_zz_stream import A, ENV_KEYS, KINDS, L, MD, R, S

pytestmark = pytest.mark.gpu

W = 16
FP16_KINDS = ["lat_cluster", "tc", "stream_fp16"]
# per stream: (frames, prompt samples or None, open step); stream 7's frames never cover its prompt
STREAMS = [(30, None, 0), (12, 23, 0), (25, 7, 0), (20, 41, 0), (16, 13, 0), (22, 52, 0), (22, 3, 4), (6, 60, 0)]
SEEDS = [0x7000 + i for i in range(len(STREAMS))]


def _env(kind, monkeypatch):
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    for k, v in KINDS[kind][1].items():
        monkeypatch.setenv(k, v)


def _cond(frames, net):
    import torch
    return torch.from_numpy(np.ascontiguousarray(_host(frames, net)[:, :, None].transpose(3, 2, 1, 0))).cuda()


def _serve(pool, frames, prompts, rng):
    """The streams through the pool: pushes of 0 to 3 frames per step; stream 1's prompt frames arrive over several pushes; streams 4
    and 5 get 12 frames at step 1, so prompts of 13 and 52 samples become scoreable in one step; stream 2 stalls for steps 3 .. 8;
    stream 6 opens at step 4.  Returns each stream's concatenated samples."""
    import torch
    n = len(STREAMS)
    ids, got, given = {}, {}, [0] * n
    for step in range(400):
        for j, (T, _, opened) in enumerate(STREAMS):
            if step < opened:
                continue
            if j not in ids:
                ids[j] = pool.open(SEEDS[j], prompts[j])
            if j == 2 and 3 <= step < 8 or j in (4, 5) and step == 0:
                continue
            k = 12 if j in (4, 5) and step == 1 else int(rng.integers(0, 4))
            k = min(k, T - given[j])
            if k:
                piece = frames[j][:, given[j]:given[j] + k]
                pool.push(ids[j], torch.from_numpy(piece).cuda() if step % 2 else piece)
                given[j] += k
            elif given[j] == T and ids[j] in pool._streams and not pool._streams[ids[j]].finished:
                pool.finish(ids[j])
        for i, y in pool.step().items():
            got.setdefault(i, []).append(y.cpu().numpy())
        if len(ids) == n and not pool._streams:
            break
    assert not pool._streams
    return [np.concatenate(got[ids[j]]) if ids[j] in got else np.empty(0, np.int32) for j in range(n)]


@pytest.mark.parametrize("kind", FP16_KINDS)
def test_prompted_pool_streams_equal_infer(kind, monkeypatch):
    import torch
    from nv_wavenet_b200.nv_wavenet import Impl
    rng = np.random.default_rng(191)
    net = _network(rng)
    frames = [rng.standard_normal((CC, T)).astype(np.float32) for T, _, _ in STREAMS]
    prompts = [None if P is None else torch.from_numpy(rng.integers(0, A, P).astype(np.int32)) for _, P, _ in STREAMS]
    _env(kind, monkeypatch)
    wnet = _net(refgen.lively_inputs(67, R, S, A, L, 1, 1), L, R, S, A, MD)
    pool = wnet.open_live_pool(*[torch.from_numpy(a) for a in net], STRIDE, KINDS[kind][2], W, fp16=True)
    groups = []
    score_group = pool._score_group
    pool._score_group = lambda g: (groups.append([P for _, P in g]), score_group(g))[1]
    got = _serve(pool, frames, prompts, np.random.default_rng(6))
    assert any(13 in g and 52 in g for g in groups), groups              # two prompts of different lengths, one scoring stream
    assert pool.resumes > 0 and pool.launches > 0
    pool.close()
    for j, (T, P, _) in enumerate(STREAMS):
        if P is not None and P >= T * STRIDE:
            assert got[j].size == 0, j
            continue
        want = wnet.infer(_cond(frames[j], net), Impl.AUTO, seed=SEEDS[j], fp16=True,
                          prompt=None if P is None else prompts[j][None]).cpu().numpy()[0, P or 0:]
        assert np.array_equal(got[j], want), (kind, j, got[j].shape, want.shape, np.argwhere(got[j] != want[:got[j].size])[:5])


@pytest.mark.parametrize("kind", FP16_KINDS)
def test_open_live_prompt_equals_infer(kind, monkeypatch):
    """Pushes of 0, 1, 1, 4, 3, 15 (more than the ring), 2 and 14 frames with a prompt of 61 samples, which spans scoring pieces of
    several pushes and crosses the window of 24: the pushes give infer(prompt=)[:, 61:] of the finished frames, bit for bit."""
    import torch
    from nv_wavenet_b200.nv_wavenet import Impl
    rng = np.random.default_rng(193)
    net = _network(rng)
    B, P, Wl = KINDS[kind][2], 61, 24
    sizes = [0, 1, 1, 4, 3, 15, 2, 14]
    frames = rng.standard_normal((B, CC, sum(sizes))).astype(np.float32)
    prompt = torch.from_numpy(rng.integers(0, A, (B, P)).astype(np.int32))
    _env(kind, monkeypatch)
    wnet = _net(refgen.lively_inputs(71, R, S, A, L, 1, 1), L, R, S, A, MD)
    live = wnet.open_live(*net, STRIDE, B, 0xBEEF, window=Wl, fp16=True, prompt=prompt)
    ys, a = [], 0
    for k in sizes:
        ys.append(live.push(frames[:, :, a:a + k]).cpu().numpy())
        a += k
    live.close()
    got = np.concatenate(ys, axis=1)
    cond = torch.from_numpy(np.ascontiguousarray(np.stack([_host(frames[b], net) for b in range(B)], axis=2).transpose(3, 2, 1, 0))).cuda()
    want = wnet.infer(cond, Impl.AUTO, seed=0xBEEF, fp16=True, window=Wl, prompt=prompt).cpu().numpy()[:, P:]
    assert got.shape == want.shape and np.array_equal(got, want), (kind, np.argwhere(got != want)[:5])


@pytest.mark.parametrize("kind", FP16_KINDS)
def test_scorer_state_resumes_in_another_engine(kind, monkeypatch):
    """Prompts of 6 and 29 samples scored in rows 0 and 1 of a scoring stream of a 5-row engine of window 16 (64 rows for the
    tensor-core kernel); their states load into slots 0 and 3 of an engine of another batch and window 24 at t0 = 24, next to
    other utterances, and continue as infer(prompt=) does."""
    import torch
    from nv_wavenet_b200.nv_wavenet import Impl
    w = refgen.lively_inputs(67, R, S, A, L, 1, 1)
    w = dict(w, Bzs=np.zeros_like(w["Bzs"]), Bza=np.zeros_like(w["Bza"]))            # NVWaveNet has no output biases
    rng = np.random.default_rng(197)
    Ps, n, seeds = [6, 29], 90, [0x51, 0x52]
    lhs = [refgen.lively_inputs(300 + j, R, S, A, L, 1, n)["Lh"][:, :, 0] for j in range(2)]          # [n][L][2R]
    prompts = [rng.integers(0, A, P).astype(np.int32) for P in Ps]
    B1 = KINDS[kind][2]
    e1 = _make(kind, B1, W, monkeypatch)
    e1.load(w)
    codes = np.full((2, max(Ps)), 128, np.int32)
    for j, p in enumerate(prompts):
        codes[j, :len(p)] = p
    states = [None, None]
    a = 0
    for end in sorted(Ps):
        while a < end:
            m = min(end - a, W - a % W)
            lh = np.zeros((m, L, B1, 2 * R), np.float32)
            for j in range(2):
                e = min(Ps[j], a + m)
                if e > a:
                    lh[:e - a, :, j] = lhs[j][a:e]
            e1.set_conditioning(lh, a % W, m)
            e1.score_stream(codes[:, a:a + m], a)
            a += m
        j = Ps.index(end)
        states[j] = e1.score_save_states([j], [seeds[j]])
    e1.close()

    B2, W2 = (128 if kind == "tc" else 8), 24
    r = _Run(_make(kind, B2, W2, monkeypatch), w)
    for b in range(B2):
        r.start(b, refgen.lively_inputs(400 + b % 7, R, S, A, L, 1, 120)["Lh"][:, :, 0], 900 + b)
    r.run(W2)
    r.load(3, lhs[1], states[1], Ps[1])
    r.load(0, lhs[0], states[0], Ps[0])
    out = [r.run(W2) for _ in range(4)]
    r.e.close()
    wnet = _net(w, L, R, S, A, MD)
    for j, slot in ((0, 0), (1, 3)):
        cond = torch.from_numpy(np.ascontiguousarray(lhs[j][:, :, None].transpose(3, 2, 1, 0))).cuda()
        want = wnet.infer(cond, Impl.AUTO, seed=seeds[j], fp16=True, prompt=torch.from_numpy(prompts[j])[None]).cpu().numpy()[0, Ps[j]:]
        got = np.concatenate([o[slot] for o in out])[:n - Ps[j]]
        assert np.array_equal(got, want[:got.size]), (kind, j, np.argwhere(got != want[:got.size])[:5])
