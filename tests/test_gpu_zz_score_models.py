"""Scoring by model (nvwn_set_score_models, ModelSet.log_likelihood / log_likelihood_many / infer_many(prompts=)): every scoring
row of an engine holding several models gives, bit for bit, the logp, logits and slot state a one-model engine of its model gives
the same utterance -- on every fp16 engine kind, R 32 / 64 / 128, any table, fewer rows than the engine, windowed streams whose
chunks wrap the store, packed queues and prompted generation; an all-zero table is the one-model scorer; every refusal changes
nothing."""
import numpy as np
import pytest

from tests import refgen
from tests.test_gpu_zz_models import _nets
from tests.test_gpu_zz_stream import A, ENV_KEYS, S

pytestmark = pytest.mark.gpu

L, MD = 8, 16
SEEDS = [0x61, 0x62, 0x63]                                   # weights of models 0 .. 2
ENVS = {"lat_cluster": {"NVWN_FP16_KERNEL": "lat"}, "lat_single": {"NVWN_FP16_KERNEL": "lat", "NVWN_LAT_CLUSTER": "0"},
        "tc": {"NVWN_FP16_KERNEL": "tc"}, "stream_fp16": {"NVWN_FP16_KERNEL": "stream"}}


def _set_env(kind, monkeypatch):
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    for k, v in ENVS.get(kind, {}).items():
        monkeypatch.setenv(k, v)


def _fresh(w, R, B, N, lh, S_=S):
    import nv_wavenet_b200 as nw
    e = nw.NVWavenetInfer(L, MD, B, N, R=R, S=S_, A=A, dtype=nw.FP16)
    e.load(w)
    e.set_conditioning_stream(np.ascontiguousarray(lh[:N]), 0)
    return e


def _setup(kind, R, B, N, monkeypatch, models=3, S_=S):
    """weights per model, conditioning [N][L][B][2R], an engine holding model m as m (donors freed), and one per-model engine each"""
    _set_env(kind, monkeypatch)
    ws = [refgen.lively_inputs(s, R, S_, A, L, B, N) for s in SEEDS[:models]]
    lh = ws[0]["Lh"]
    e = _fresh(ws[0], R, B, N, lh, S_)
    for m in range(1, models):
        d = _fresh(ws[m], R, 4, 3, lh[:, :, :4], S_)
        e.set_model(m, d)
        d.close()
    return ws, lh, e, [_fresh(w, R, B, N, lh, S_) for w in ws]


def _tables(B, rng):
    return {"one": [2] * B, "alternate": [b % 3 for b in range(B)], "scattered": [int(v) for v in rng.choice([0, 1, 2], B, p=[.2, .3, .5])],
            "single": [1 if b == B // 2 else 0 for b in range(B)]}


def _same(got, want, rows, what):
    for b in rows:
        assert np.array_equal(got[b].view(np.uint32), want[b].view(np.uint32)), (what, b)


@pytest.mark.parametrize("kind,R,S_,B", [("lat_cluster", 64, S, 37), ("lat_single", 64, S, 37), ("tc", 64, S, 128),
                                         ("stream_fp16", 64, S, 37), ("auto", 32, 128, 70), ("auto", 128, S, 70)])
def test_mixed_tables_match_per_model_engines(kind, R, S_, B, monkeypatch):
    N = 300                                                   # chunks of 16384 / B steps: several per call at B = 128
    ws, lh, e, refs = _setup(kind, R, B, N, monkeypatch, S_=S_)
    audio = np.random.default_rng(3).integers(0, A, (B, N)).astype(np.int32)
    want = [r.score(audio, logits=True) for r in refs]
    assert not np.array_equal(want[0][0], want[1][0])
    for name, table in _tables(B, np.random.default_rng(4)).items():
        e.set_score_models(table)
        lp, lg = e.score(audio, logits=True)
        for m in range(3):
            rows = [b for b in range(B) if table[b] == m]
            _same(lp, want[m][0], rows, (name, "logp", m))
            _same(lg, want[m][1], rows, (name, "logits", m))
        # fewer rows than the engine: entries [0, Bs) of the table
        Bs = B - 5
        lp, lg = e.score(audio[:Bs], batch_size=Bs, logits=True)
        for m in range(3):
            rows = [b for b in range(Bs) if table[b] == m]
            _same(lp, want[m][0], rows, (name, "Bs", m))
            _same(lg, want[m][1], rows, (name, "Bs logits", m))
    for r in refs + [e]:
        r.close()


@pytest.mark.parametrize("kind", ["lat_cluster", "tc"])
def test_windowed_stream_wrapping_the_store(kind, monkeypatch):
    """A stream of 700 samples through an engine of 300 in windows of 250, 300 and 150 samples: chunks end inside windows and
    windows wrap the store; every row equals one whole-length call on its model's engine."""
    R, B, N, total = 64, 64, 300, 700                         # chunks of 256 steps
    _set_env(kind, monkeypatch)
    ws = [refgen.lively_inputs(s, R, S, A, L, B, total) for s in SEEDS]
    lh = ws[0]["Lh"]
    e = _fresh(ws[0], R, B, N, lh)
    for m in (1, 2):
        d = _fresh(ws[m], R, 4, 3, lh[:, :, :4])
        e.set_model(m, d)
        d.close()
    audio = np.random.default_rng(5).integers(0, A, (B, total)).astype(np.int32)
    table = _tables(B, np.random.default_rng(6))["scattered"]
    e.set_score_models(table)
    lp = np.zeros((B, total), np.float32)
    first = 0
    for n in (250, 300, 150):
        e.set_conditioning_stream(np.ascontiguousarray(lh[first:first + n]), first)
        lp[:, first:first + n] = e.score_stream(audio[:, first:first + n], first)
        first += n
    for m in range(3):
        ref = _fresh(ws[m], R, B, total, lh)
        want = ref.score(audio)
        _same(lp, want, [b for b in range(B) if table[b] == m], m)
        ref.close()
    e.close()


def test_states_zero_table_and_refusals(monkeypatch):
    import nv_wavenet_b200 as nw
    R, B, N = 64, 20, 40
    ws, lh, e, refs = _setup("lat_cluster", R, B, N, monkeypatch)
    audio = np.random.default_rng(7).integers(0, A, (B, N)).astype(np.int32)
    plain = refs[0].score(audio, logits=True)
    # an all-zero table is the one-model scorer
    e.set_score_models([0] * B)
    z = e.score(audio, logits=True)
    _same(z[0], plain[0], range(B), "zero logp")
    _same(z[1], plain[1], range(B), "zero logits")
    # slot states of scored rows: byte for byte those of the row's model's engine
    table = [b % 3 for b in range(B)]
    e.set_score_models(table)
    e.score_stream(audio[:, :29], 0)
    for r in refs:
        r.score_stream(audio[:, :29], 0)
    rows = [4, 0, 11, 7]
    got = e.score_save_states(rows, seeds=[9, 8, 7, 6]).cpu().numpy()
    for i, b in enumerate(rows):
        want = refs[table[b]].score_save_states([b], seeds=[9 - i]).cpu().numpy()
        assert np.array_equal(got[i], want[0]), b
    # refusals change nothing: the table, and the stream they would continue
    bad = lambda: pytest.raises(nw.NvwnError, match=r"code -1\)")
    for t in ([0] * (B - 1), [0] * (B + 1), [-1] + [0] * (B - 1), [nw.infer.MAX_MODELS] + [0] * (B - 1), [5] + [0] * (B - 1)):
        with bad():
            e.set_score_models(t)
    more = e.score_stream(audio[:, 29:], 29)                  # the stream is still open, on the same table
    for m in range(3):
        _same(more, refs[m].score_stream(audio[:, 29:], 29), [b for b in range(B) if table[b] == m], ("continued", m))
    e.set_score_models(table)                                 # a new table ends the stream
    with bad():
        e.score_stream(audio[:, :5], 40)
    # a prime whose row was scored with another model than its slot's group runs
    G = e.model_group
    e.set_group_models([1] + [0] * ((B - 1) // G))
    e.set_score_models([1] * G + [2] * (B - G))
    e.reset_history()
    e.score_stream(audio[:, :6], 0)
    with bad():
        e.prime_from_score()                                  # rows of groups 1 and 2 were scored with model 2
    with bad():
        e.prime_slots_from_score([0, G], [1, G + 1])          # row G (model 2) into group 1 (model 0)
    e.prime_slots_from_score([0, 1], [2, 3])                  # model 1 rows into group 0 (model 1): accepted
    # set_model(m, other) repacks model m's image, and ends a stream whose rows run it
    d = _fresh(ws[0], R, 4, 3, lh[:, :, :4])
    e.set_model(2, d)
    d.close()
    with bad():
        e.score_stream(audio[:, 6:8], 6)
    e.set_score_models([2] * B)
    again = e.score(audio, logits=True)
    _same(again[0], plain[0], range(B), "repacked logp")
    _same(again[1], plain[1], range(B), "repacked logits")
    for r in refs + [e]:
        r.close()


def _conds(lengths, R, seed):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [0.5 * torch.randn((2 * R, L, n), generator=g, device="cuda") for n in lengths]


def test_modelset_log_likelihood(monkeypatch):
    import torch
    from nv_wavenet_b200.nv_wavenet import ModelSet
    _set_env("auto", monkeypatch)
    R = 64
    nets = _nets(L, MD, 3)
    B, N = 9, 500
    cond = _conds([N] * B, R, 11)
    cond = torch.stack(cond, dim=1).contiguous()              # [2R][B][L][N]
    audio = torch.randint(0, A, (B, N), dtype=torch.int32, device="cuda", generator=torch.Generator(device="cuda").manual_seed(12))
    models = [2, 0, 1, 1, 2, 0, 2, 2, 1]
    ms = ModelSet(nets)
    for window in (None, 128):
        got = ms.log_likelihood(models, cond, audio, window=window).cpu().numpy()
        for b in range(B):
            want = nets[models[b]].log_likelihood(cond[:, b:b + 1].contiguous(), audio[b:b + 1], window=window)[0].cpu().numpy()
            assert np.array_equal(got[b].view(np.uint32), want.view(np.uint32)), (window, b)
    ms.close()


def test_modelset_log_likelihood_many(monkeypatch):
    from nv_wavenet_b200.nv_wavenet import ModelSet
    import torch
    _set_env("auto", monkeypatch)
    R = 64
    nets = _nets(L, MD, 3)
    rng = np.random.default_rng(21)
    n = 24
    lengths = [int(v) for v in rng.integers(20, 700, n)]
    models = [int(v) for v in rng.integers(0, 3, n)]
    conds = _conds(lengths, R, 22)
    audios = [torch.from_numpy(rng.integers(0, A, m).astype(np.int32)) for m in lengths]
    ms = ModelSet(nets)
    got = ms.log_likelihood_many(models, conds, audios, slots=8, window=256)
    for u in range(n):
        want = nets[models[u]].log_likelihood_many([conds[u]], [audios[u]], slots=1, window=256)[0].cpu().numpy()
        assert np.array_equal(got[u].cpu().numpy().view(np.uint32), want.view(np.uint32)), (u, models[u])
    with pytest.raises(ValueError, match="distinct models"):
        ms.log_likelihood_many(models, conds, audios, slots=2, window=256)
    ms.close()


def test_modelset_infer_many_prompts(monkeypatch):
    import torch
    from nv_wavenet_b200.nv_wavenet import Impl, ModelSet
    _set_env("auto", monkeypatch)
    R = 64
    nets = _nets(L, MD, 3)
    rng = np.random.default_rng(31)
    n = 14
    lengths = [int(v) for v in rng.integers(60, 300, n)]
    models = [int(v) for v in rng.integers(0, 3, n)]
    seeds = [int(v) for v in rng.integers(0, 2 ** 62, n)]
    prompts = [None if u % 4 == 3 else torch.from_numpy(rng.integers(0, A, int(rng.integers(1, lengths[u] // 2))).astype(np.int32))
               for u in range(n)]
    conds = _conds(lengths, R, 32)
    ms = ModelSet(nets)
    timing = {}
    got = ms.infer_many(models, conds, seeds, slots=16, window=64, fp16=True, timing=timing, prompts=prompts)
    assert timing["prime_s"] > 0
    for u in range(n):
        want = nets[models[u]].infer(conds[u][:, None].contiguous(), Impl.AUTO, seed=seeds[u], fp16=True, prompt=None if prompts[u] is None
                                     else prompts[u][None])[0].cpu().numpy()
        assert np.array_equal(got[u].cpu().numpy(), want), (u, models[u], np.argwhere(got[u].cpu().numpy() != want)[:5])
    ms.close()
