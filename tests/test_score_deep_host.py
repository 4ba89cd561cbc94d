"""The reach of tests/test_gpu_zz_score_deep.py, recomputed without a GPU from the scorer's chunk rule.

The scorer runs a call in chunks of T = min(N, max(1, SCORE_ROWS / B)) steps of the engine's B (score_range in wn_engine.cu), and a
carry of layer l after a chunk of Tc steps copies its d_l-step front in ceil(d_l / Tc) pieces.  Each GPU case is there to have the
largest dilation read across at least two carries, and some to reach more: a change to SCORE_ROWS or to a case's shape must not
silently leave them inside one chunk."""
from tests.test_gpu_zz_prime import _dils
from tests.test_gpu_zz_score_deep import (PACKED, PACKED_UTTS, PRIME, PRIME_BS, PRIME_ROWS, SCORED, carries_read, chunk_steps, chunks,
                                          score_rows)


def _pieces(d, Tc):
    return -(-d // Tc)


def test_scored_cases_read_across_carries():
    for case, (R, S, L, md, B, bs, N, rows) in SCORED.items():
        T, dmax = chunk_steps(B, N), max(_dils(L, md))
        plan = chunks(T, N)
        assert T == min(N, max(1, score_rows() // B)) and sum(Tc for _, Tc in plan) == N
        assert dmax >= 2 * T and N >= dmax + 2 * T, (case, T, dmax, N)
        assert carries_read(N - 1, dmax, T) >= 2, case
        assert plan[-1][1] < T, f"{case}: the last chunk is not ragged"
        assert max(rows) < bs <= B, case
    T = {case: chunk_steps(c[4], c[6]) for case, c in SCORED.items()}
    assert T["c3_b64"] == 256 and len(chunks(256, SCORED["c3_b64"][6])) - 1 == 4             # four carries at the serving batch
    assert T["l10_b2048"] == 8 and _pieces(512, 8) == 64                                     # a carry of d = 512 is 64 copies
    R, S, L, md, B, bs, N, _ = SCORED["c3_bs150_of_200"]
    assert bs < B and N % T["c3_bs150_of_200"] and T["c3_bs150_of_200"] == 81                # fronts at stride 150 in buffers of 200
    for case in ("r128", "r32"):
        assert T[case] == 128 and max(_dils(SCORED[case][2], SCORED[case][3])) == 2 * T[case]
    assert {SCORED[c][0] for c in SCORED} == {32, 64, 128}


def test_packed_utterances_start_before_a_boundary():
    R, S, L, md, B, N = PACKED
    T, dmax = chunk_steps(B, N), max(_dils(L, md))
    assert T == 256
    for r, s, n in PACKED_UTTS:
        assert 0 < -s % T <= 8, (r, s)                            # a few steps before a chunk boundary
        assert n > dmax and s + n <= N and r < B
        assert carries_read(s + n - 1, dmax, T) >= 2, (r, s, n)   # its last steps read x[t - 512] across two carries


def test_prime_fronts_come_from_several_carries():
    R, S, L, md, B, P, G = PRIME
    T, dmax = chunk_steps(B, P + G), max(_dils(L, md))
    plan = chunks(T, P)
    assert P > dmax + T and len(plan) == 4 and G == dmax
    # the front of d = 512 at P holds x[P - 512, P), written in chunks that are two carries apart, and the prompt's last carry
    # (after a chunk of P mod T steps) copies it in many pieces
    assert carries_read(P - 1, dmax, T) >= 2 and _pieces(dmax, plan[-1][1]) == 57
    assert max(PRIME_ROWS) < min(PRIME_BS.values()) and PRIME_BS["tc"] == B and all(bs < B for k, bs in PRIME_BS.items() if k != "tc")
