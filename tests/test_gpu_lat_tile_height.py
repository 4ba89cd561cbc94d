"""Tile height of the three-CTA cluster kernel: 8 utterances per cluster while all of those clusters are resident at once, else 16.
Both sides of the choice must give, bit for bit, what the single-CTA kernel (16-utterance tiles, NVWN_LAT_CLUSTER=0) gives: the
sampled indices and the last step's activations."""
import numpy as np
import pytest

import nv_wavenet_b200 as nw
from nv_wavenet_b200 import _lib
from tests import refgen

pytestmark = pytest.mark.gpu


def _run(w, L, B, N, R, S, A, md, cluster, monkeypatch):
    monkeypatch.setenv("NVWN_FP16_KERNEL", "lat")
    monkeypatch.setenv("NVWN_LAT_CLUSTER", "1" if cluster else "0")
    e = nw.NVWavenetInfer(L, md, B, N, R=R, S=S, A=A, dtype=nw.FP16)
    e.load(w); e.set_inputs(w["Lh"], w["selectors"])
    y = np.zeros((B, N), np.int32)
    e.run(N, B, y, dump_activations=True); e.synchronize()
    return y, e.activations(), e.launch_info()


def _assert_same(a, b):
    ya, acta = a[:2]
    yb, actb = b[:2]
    assert np.array_equal(ya, yb)
    assert acta.keys() == actb.keys()
    for k in acta:
        x, z = np.ascontiguousarray(acta[k]), np.ascontiguousarray(actb[k])
        assert x.shape == z.shape and np.array_equal(x.view(np.uint32), z.view(np.uint32)), k


@pytest.mark.parametrize("S, L, md", [(256, 20, 16), (128, 20, 16), (256, 12, 1)])
def test_eight_row_clusters_equal_single_cta(S, L, md, monkeypatch):
    """B = 13: two 8-row clusters, the second one ragged, both halves of one 16-row store tile.  L = 12 with maxDil = 1 is the
    shortest distance (24 steps) between the prep CTA's two reads of one history-ring row, the chain CTA rewriting it in between."""
    R, A, B, N = 64, 256, 13, 80
    w = refgen.lively_inputs(31 + S, R, S, A, L, B, N)
    clu = _run(w, L, B, N, R, S, A, md, True, monkeypatch)
    one = _run(w, L, B, N, R, S, A, md, False, monkeypatch)
    assert clu[2]["cluster"] == 3 and clu[2]["batch_per_cta"] == 8 and clu[2]["grid"] == 3 * 2
    assert one[2]["cluster"] == 1 and one[2]["batch_per_cta"] == 16
    _assert_same(clu, one)
    assert len(np.unique(clu[0])) > 8


def test_sixteen_row_clusters_past_the_eight_row_limit(monkeypatch):
    """400 utterances: more 8-row clusters than an H100 keeps resident (about 45), so the 16-row cluster runs (25 clusters)."""
    R, S, A, L, B, N, md = 64, 256, 256, 12, 400, 200, 64
    fit8, fit16 = (_lib.lib().nvwn_debug_lat_max_clusters(S, rows) for rows in (8, 16))
    if not (fit8 < (B + 7) // 8 and (B + 15) // 16 <= fit16):
        pytest.skip(f"{fit8} / {fit16} resident 8- / 16-row clusters: 400 utterances do not fall between the two limits on this device")
    w = refgen.lively_inputs(47, R, S, A, L, B, N)
    clu = _run(w, L, B, N, R, S, A, md, True, monkeypatch)
    one = _run(w, L, B, N, R, S, A, md, False, monkeypatch)
    assert clu[2]["cluster"] == 3 and clu[2]["batch_per_cta"] == 16 and clu[2]["grid"] == 3 * 25
    _assert_same(clu, one)
