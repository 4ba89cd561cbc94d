"""Multi-model serving (nvwn_set_model, nvwn_set_group_models, ModelSet): every row of an engine holding several models generates
exactly what a one-model engine of its model generates -- samples and last-step dumps -- on every kernel, through table changes,
restarts, parks and resumes; the donor is copied, not referenced; every refusal changes nothing."""
import numpy as np
import pytest

from tests import refgen
from tests.common import bits_equal
from tests.test_gpu_zz_selectors import _net
from tests.test_gpu_zz_stream import A, ENV_KEYS, KINDS, R, S

pytestmark = pytest.mark.gpu

L, MD, T = 12, 8, 40
SEEDS = [0x51, 0x52, 0x53, 0x54]        # weights of models 0 .. 3


def _max8():
    from nv_wavenet_b200 import _lib
    return _lib.lib().nvwn_debug_lat_max_clusters(S, 8)


# kind -> (KINDS entry, batch: several groups, the last one partial, expected launch info)
def _kinds():
    out = {k: (k, B, KINDS[k][3]) for k, B in (("lat_cluster", 20), ("lat_single", 37), ("tc", 160), ("stream_fp16", 10), ("fp32", 10),
                                                ("fp32_fast", 10))}
    out["lat_cluster16"] = ("lat_cluster", None, {"kernel": 18, "cluster": 3, "batch_per_cta": 16})
    return out


MKINDS = _kinds()


def _batch(kind):
    B = MKINDS[kind][1]
    return B if B is not None else _max8() * 8 + 1           # just past what 8-row clusters serve at once


def _eng(kind, B, n, monkeypatch):
    import nv_wavenet_b200 as nw
    dt, env, _, _ = KINDS[MKINDS[kind][0]]
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    dtype = {"fp16": nw.FP16, "fp32": nw.FP32, "fp32_fast": nw.FP32_FAST}[dt]
    return nw.NVWavenetInfer(L, MD, B, n, R=R, S=S, A=A, dtype=dtype)


def _weights(B, n=T):
    return [refgen.lively_inputs(s, R, S, A, L, B, n) for s in SEEDS]


def _engine_with_models(kind, B, W, ws, monkeypatch):
    """An engine whose model 0 is ws[0] and model m is ws[m], copied from donors of another batch and length that are then freed."""
    e = _eng(kind, B, W, monkeypatch)
    e.load(ws[0])
    for m, w in enumerate(ws[1:], 1):
        d = _eng(kind, 4, 3, monkeypatch)
        d.load(w)
        e.set_model(m, d)
        d.close()
    return e


def _ranges(W, breaks, total=T):
    """uneven launch ranges of at most W samples (crossing the wrap of a W-sample engine) that end at every time in `breaks`"""
    sizes = [W, max(1, W - 2), 1, W, (W + 1) // 2, 2]
    out, first, i = [], 0, 0
    while first < total:
        nxt = min([first + sizes[i % len(sizes)], total] + [t for t in breaks if t > first])
        out.append((first, nxt - first))
        first, i = nxt, i + 1
    return out


def _generate(e, lh, seeds, W, tables=None, restarts=None, total=T, pause=None):
    """Every slot starts at 0 with seeds[b]; then launches over _ranges.  tables: {t: table set before the launch at t};
    restarts: {t: [(slot, seed, cond [total - t][L][2R])]}; pause: (t, hook(e)) run before the launch at t.  Conditioning by
    slot, selectors by slot.  Returns samples [B][total] and the last step's dumps."""
    tables, restarts = tables or {}, restarts or {}
    B = e.B
    lh = lh.copy()
    e.reset_history()
    e.restart_slots(range(B), seeds)
    y = np.zeros((B, total), np.int32)
    breaks = set(tables) | set(restarts) | ({pause[0]} if pause else set())
    for first, n in _ranges(W, breaks, total):
        if first in tables:
            e.set_group_models(tables[first])
        if first in restarts:
            e.restart_slots([s for s, _, _ in restarts[first]], [sd for _, sd, _ in restarts[first]])
            for s, _, c in restarts[first]:
                lh[first:, :, s] = c
        if pause and pause[0] == first:
            pause[1](e, lh)
        e.set_conditioning_slots(np.ascontiguousarray(lh[first:first + n]), range(B), first)
        e.set_selectors_random_slots(first, n)
        e.run_stream(first, n, B, dump_activations=(first + n == total))
        e.get_yout_stream(y[:, first:first + n], first, n)
    e.synchronize()
    return y, e.activations()


def _same_row(got, want, b):
    yg, ag = got
    yw, aw = want
    assert np.array_equal(yg[b], yw[b]), (b, np.argwhere(yg[b] != yw[b])[:5])
    for k, axis in (("xt", 1), ("skip", 1), ("zs", 0), ("za", 0), ("p", 0)):
        assert bits_equal(np.take(ag[k], [b], axis=axis), np.take(aw[k], [b], axis=axis)), (b, k)


def _table(n_groups, pattern):
    return [pattern[g % len(pattern)] for g in range(n_groups)]


@pytest.mark.parametrize("kind", sorted(MKINDS))
def test_rows_match_a_one_model_engine(kind, monkeypatch):
    B = _batch(kind)
    total = 24 if kind == "lat_cluster16" else T
    ws = _weights(B, total)[:3]
    W = 7
    seeds = [0x900 + 3 * b for b in range(B)]
    e = _engine_with_models(kind, B, W, ws, monkeypatch)
    G = e.model_group
    n_groups = (B + G - 1) // G
    assert n_groups >= 3 and B % G != 0
    table = _table(n_groups, [2, 0, 1, 1, 2])
    got = _generate(e, ws[0]["Lh"], seeds, W, tables={0: table}, total=total)
    info = e.launch_info()
    assert all(info[k] == v for k, v in MKINDS[kind][2].items()), info
    if kind == "lat_cluster":
        assert G == 8 and info["batch_per_cta"] == 8
    if kind == "lat_cluster16":
        assert G == 16
    assert len(np.unique(got[0])) > 8
    wants = {m: _generate(_eng_loaded(kind, B, W, ws[m], monkeypatch), ws[0]["Lh"], seeds, W, total=total) for m in range(3)}
    for m in range(3):
        rows = [b for b in range(B) if table[b // G] == m]
        assert rows
        for b in rows:
            _same_row(got, wants[m], b)
        if m:                                                    # the models differ where it shows
            assert not np.array_equal(got[0][rows], wants[0][0][rows])


def _eng_loaded(kind, B, W, w, monkeypatch):
    e = _eng(kind, B, W, monkeypatch)
    e.load(w)
    return e


@pytest.mark.parametrize("kind", ["lat_cluster", "lat_single", "tc", "stream_fp16", "fp32"])
def test_table_change_between_windows(kind, monkeypatch):
    B = _batch(kind)
    ws = _weights(B)[:3]
    W, tc = 7, 17
    seeds = [0x700 + b for b in range(B)]
    rng = np.random.default_rng(5)
    e = _engine_with_models(kind, B, W, ws, monkeypatch)
    G = e.model_group
    n_groups = (B + G - 1) // G
    t1 = _table(n_groups, [0, 1, 2])
    t2 = list(t1)
    t2[1] = 2                                                    # group 1 switches from model 1 to model 2 at tc
    switched = list(range(G, min(B, 2 * G)))
    cond = {s: (0.5 * rng.standard_normal((T - tc, L, 2 * R))).astype(np.float32) for s in switched}
    new_seeds = {s: 0xABC00 + s for s in switched}
    got = _generate(e, ws[0]["Lh"], seeds, W, tables={0: t1, tc: t2}, restarts={tc: [(s, new_seeds[s], cond[s]) for s in switched]})
    still = _generate(e, ws[0]["Lh"], seeds, W, tables={0: t1})
    for b in range(B):
        if b not in switched:
            _same_row(got, still, b)
    # a restarted row equals a fresh one-model engine of model 2 started with its utterance in that slot
    fresh = _eng_loaded(kind, B, W, ws[2], monkeypatch)
    lh = ws[0]["Lh"].copy()
    for s in switched:
        lh[:T - tc, :, s] = cond[s]
    want = _generate(fresh, lh, [new_seeds.get(b, 0) for b in range(B)], W, total=T - tc)[0]
    for s in switched:
        assert np.array_equal(got[0][s, tc:], want[s]), (s, np.argwhere(got[0][s, tc:] != want[s])[:5])


@pytest.mark.parametrize("kind", ["lat_cluster", "tc", "stream_fp16"])
def test_model_is_a_copy(kind, monkeypatch):
    B = _batch(kind)
    ws = _weights(B)
    W = 9
    seeds = list(range(1, B + 1))
    e = _eng_loaded(kind, B, W, ws[0], monkeypatch)
    donor = _eng_loaded(kind, 4, 3, ws[1], monkeypatch)
    e.set_model(1, donor)
    n_groups = (B + e.model_group - 1) // e.model_group
    table = _table(n_groups, [1, 0])
    rows1 = [b for b in range(B) if table[b // e.model_group] == 1]
    rows0 = [b for b in range(B) if table[b // e.model_group] == 0]
    ref = {i: _generate(_eng_loaded(kind, B, W, ws[i], monkeypatch), ws[0]["Lh"], seeds, W) for i in range(4)}

    def check(want1, want0):
        got = _generate(e, ws[0]["Lh"], seeds, W, tables={0: table})
        for b in rows1:
            _same_row(got, ref[want1], b)
        for b in rows0:
            _same_row(got, ref[want0], b)

    check(1, 0)
    donor.load(ws[2])                                            # the donor changes: the model does not
    check(1, 0)
    e.set_model(1, donor)                                        # set again: it does
    check(2, 0)
    e.load(ws[3])                                                # model 0 through the setters: model 1's rows stay
    check(2, 3)
    donor.close()
    check(2, 3)


def test_park_and_resume_across_groups(monkeypatch):
    kind, B, W, tp = "lat_cluster", 20, 7, 19
    ws = _weights(B)[:2]
    seeds = [0x300 + b for b in range(B)]
    e = _engine_with_models(kind, B, W, ws, monkeypatch)
    G = e.model_group
    table = [1, 0, 1]
    src, dst = 3, 2 * G + 1                                      # group 0 -> group 2, both model 1
    assert table[src // G] == table[dst // G] == 1
    whole = _generate(e, ws[0]["Lh"], seeds, W, tables={0: table})

    def move(eng, lh):
        state = eng.save_slots([src])
        eng.load_slots([dst], state)
        lh[tp:, :, dst] = lh[tp:, :, src]

    moved = _generate(e, ws[0]["Lh"], seeds, W, tables={0: table}, pause=(tp, move))
    assert np.array_equal(moved[0][dst, tp:], whole[0][src, tp:]), np.argwhere(moved[0][dst, tp:] != whole[0][src, tp:])[:5]
    assert bits_equal(moved[1]["za"][dst], whole[1]["za"][src])
    assert np.array_equal(moved[0][src], whole[0][src])


def test_refusals_change_nothing(monkeypatch):
    import nv_wavenet_b200 as nw
    import torch
    kind, B, W = "lat_cluster", 20, 9
    ws = _weights(B)[:2]
    seeds = [0x100 + b for b in range(B)]
    e = _engine_with_models(kind, B, W, ws, monkeypatch)
    twin = _engine_with_models(kind, B, W, ws, monkeypatch)
    G = e.model_group
    table = [1, 0, 0]
    e.set_group_models(table)
    bad = lambda: pytest.raises(nw.NvwnError, match=r"code -1\)")
    other_L = nw.NVWavenetInfer(L + 1, MD, 4, 3, R=R, S=S, A=A, dtype=nw.FP16)
    other_md = nw.NVWavenetInfer(L, 2 * MD, 4, 3, R=R, S=S, A=A, dtype=nw.FP16)
    other_dt = nw.NVWavenetInfer(L, MD, 4, 3, R=R, S=S, A=A, dtype=nw.FP32)
    other_tanh = nw.NVWavenetInfer(L, MD, 4, 3, 0, False, R=R, S=S, A=A, dtype=nw.FP16)
    for src in (other_L, other_md, other_dt, other_tanh):
        with bad():
            e.set_model(1, src)
    same = _eng_loaded(kind, 4, 3, ws[0], monkeypatch)
    for m in (0, -1, nw.infer.MAX_MODELS):
        with bad():
            e.set_model(m, same)
    for t in ([1, 0], [1, 0, 0, 0], [1, 0, 5], [1, 0, nw.infer.MAX_MODELS], [-1, 0, 0]):
        with bad():
            e.set_group_models(t)
    # primes: scoring runs model 0, so rows and slots of group 0 (model 1) are refused
    e.reset_history()
    e.set_conditioning(np.ascontiguousarray(ws[0]["Lh"][:4]), 0, 4)
    e.score_stream(torch.full((B, 4), 128, dtype=torch.int32, device="cuda"), 0)
    with bad():
        e.prime_from_score()
    with bad():
        e.prime_slots_from_score([0, 1], [G + 1, 1])
    got = _generate(e, ws[0]["Lh"], seeds, W)                  # the table set before the refused calls
    want = _generate(twin, ws[0]["Lh"], seeds, W, tables={0: table})
    assert np.array_equal(got[0], want[0])
    for k in ("xt", "skip", "zs", "za", "p"):
        assert bits_equal(got[1][k], want[1][k]), k
    for x in (other_L, other_md, other_dt, other_tanh, same):
        x.close()


def _nets(L_, md, n):
    return [_net(refgen.lively_inputs(s, R, S, A, L_, 1, 1), L_, R, S, A, md) for s in SEEDS[:n]]


@pytest.mark.parametrize("fp16", [True, False])
def test_modelset_infer_many(fp16, monkeypatch):
    import torch
    from nv_wavenet_b200.nv_wavenet import Impl, ModelSet
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    nets = _nets(L, MD, 3)
    rng = np.random.default_rng(91)
    n = 20
    lengths = [int(v) for v in rng.integers(30, 400, n)]
    models = [int(v) for v in rng.integers(0, 3, n)]
    seeds = [int(v) for v in rng.integers(0, 2 ** 62, n)]
    g = torch.Generator(device="cuda").manual_seed(92)
    conds = [0.5 * torch.randn((2 * R, L, m), generator=g, device="cuda") for m in lengths]
    ms = ModelSet(nets)
    got = ms.infer_many(models, conds, seeds, slots=16, window=64, fp16=fp16)
    for u in range(n):
        want = nets[models[u]].infer(conds[u][:, None].contiguous(), Impl.AUTO, seed=seeds[u], fp16=fp16)[0].cpu().numpy()
        assert np.array_equal(got[u].cpu().numpy(), want), (u, models[u], np.argwhere(got[u].cpu().numpy() != want)[:5])
    others = [nets[(models[u] + 1) % 3].infer(conds[u][:, None].contiguous(), Impl.AUTO, seed=seeds[u], fp16=fp16)[0].cpu().numpy()
              for u in range(3)]
    assert any(not np.array_equal(got[u].cpu().numpy(), others[u]) for u in range(3))
    ms.close()


def test_modelset_infer_many_c3(monkeypatch):
    """C3 model (L20, maxDil 512), 64 slots in 8-row groups on the cluster kernel, a window of 4 096: 40 utterances of 2 000 -
    20 000 samples over three models; six of them, chosen by seed, are bit-identical to infer() of their model alone."""
    import torch
    from nv_wavenet_b200.nv_wavenet import Impl, ModelSet
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    L3, md, n = 20, 512, 40
    rng = np.random.default_rng(81)
    lengths = [int(v) for v in rng.integers(2000, 20001, n)]
    offsets = [int(v) for v in rng.integers(0, 20000, n)]
    seeds = [int(v) for v in rng.integers(0, 2 ** 62, n)]
    models = [int(v) for v in rng.integers(0, 3, n)]
    g = torch.Generator(device="cuda").manual_seed(83)
    base = 0.5 * torch.randn((2 * R, L3, 40000), generator=g, device="cuda")
    conds = [base[:, :, o:o + m] for o, m in zip(offsets, lengths)]
    nets = _nets(L3, md, 3)
    ms = ModelSet(nets)
    got = ms.infer_many(models, conds, seeds, slots=64, window=4096, fp16=True)
    eng = ms._engine(64, 4096, True)
    info = eng.launch_info()
    assert info["cluster"] == 3 and info["batch_per_cta"] == 8 and eng.model_group == 8
    for u in sorted(rng.choice(n, 6, replace=False)):
        want = nets[models[u]].infer(conds[u][:, None].contiguous(), Impl.AUTO, seed=seeds[u], fp16=True)[0].cpu().numpy()
        assert len(np.unique(want)) > 16
        assert np.array_equal(got[u].cpu().numpy(), want), (u, np.argwhere(got[u].cpu().numpy() != want)[:5])
    ms.close()
