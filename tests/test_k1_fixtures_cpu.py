"""The fixtures of tests/k1_fixtures.py deliver what they claim (CPU only, oracle): exact sums, ties and sticky bits of the
tie sums, shared score-key prefixes, host-out edges, tile positions of the shapes, and the numpy model of the Form D
arithmetic against the oracle."""
import numpy as np
import pytest

import k1_fixtures as kf


def test_tiles_and_edges():
    for tile in list(kf.TILES_K1.values()) + list(kf.TILES_KQ.values()):
        e = kf.t_edges(tile)
        assert [T - tile for T in e[:7]] == [-8, -1, 0, 1, 4, 7, 8]
        assert e[7] % tile == tile - 1 and e[8] % tile == 1          # the second tile is partial on both sides of full
    for tile in kf.TILES_K1.values():
        assert all(f % 4 == 0 and f % tile for f in kf.window_starts(tile, 4)[1:])
    for tile in kf.TILES_KQ.values():
        assert all(f % 8 == 0 and f % tile for f in kf.window_starts(tile, 8)[1:])
    assert float(kf.MAXF) == 512 - 2 ** -15 and np.nextafter(kf.MAXF, np.float32(1e9)) == np.float32(512)


@pytest.mark.parametrize("S", [0, 1, -1, (1 << 52) + 255, (1 << 65) + (1 << 12) + 1, -((1 << 70) + (1 << 17)), 1 << 63])
def test_pow2_rows_sum_exactly(orc, S):
    n = len(kf.pow2_rows(S)) + 3
    d = kf.candidate(S, n, n + 2)[None]
    assert kf.oracle_fx(d) == ([S], [n])
    assert kf.fx_model(d) == ([S], [n])


def test_tie_sums_are_ties_or_sticky(orc):
    d = kf.tie_dims()
    sums, counts = kf.oracle_fx(d)
    assert sums == kf.tie_sums() and counts == [kf.TIE_N] * len(sums)
    tie = {S: kf.is_binary64_tie(S) for S in kf.TIE_SUMS}
    assert [S for S, t in tie.items() if t] == [(1 << 53) + 1, (1 << 53) + 3, (1 << 54) + 2, (1 << 54) + 6, (1 << 65) + (1 << 12),
                                                 (1 << 65) + 3 * (1 << 12), (1 << 70) + (1 << 17)]
    # ties go to the even neighbour, a sticky bit below the cut goes up, one short of the tie goes down
    assert float((1 << 53) + 1) == 2.0 ** 53 and float((1 << 53) + 3) == 2.0 ** 53 + 4
    assert float((1 << 65) + (1 << 12)) == 2.0 ** 65 and float((1 << 65) + 3 * (1 << 12)) == 2.0 ** 65 + 2.0 ** 14
    assert float((1 << 65) + (1 << 12) + 1) == 2.0 ** 65 + 2.0 ** 13 and float((1 << 65) + (1 << 12) - 1) == 2.0 ** 65
    assert float((1 << 70) + (1 << 17) + 1) == 2.0 ** 70 + 2.0 ** 18 and float((1 << 70) + (1 << 17)) == 2.0 ** 70
    sc = kf.scores_of(sums, counts)
    assert all(sc[k] == float(S) / 2.0 ** 52 / kf.TIE_N for k, S in enumerate(sums))
    assert np.array_equal(sc[0::2], -sc[1::2])                      # negative mirrors


def test_extreme_sums_reach_the_upper_limbs(orc):
    d = kf.extreme_dims()
    sums, counts = kf.oracle_fx(d)
    assert counts == [d.shape[1]] * 3 + [9, d.shape[1]]
    assert sums[0] > 1 << 72 and sums[1] < -(1 << 72) and sums[1] == -sums[0]
    assert (1 << 64) < sums[3] < 1 << 65
    assert abs(sums[2]) < 1 << 62 and abs(sums[4]) < 1 << 63
    assert kf.fx_model(d) == (sums, counts)
    one = kf.oracle_fx(d[:1, :1])[0][0]
    assert (1 << 61) - (1 << 40) < one < 1 << 61                     # one evaluation: just inside the int64 pre-add bound
    assert 4 * one < 1 << 63


def test_huge_sums_near_2_83(orc):
    d = kf.huge_dims(1 << 16)                                        # the same rows, shorter: the sum is linear in T
    sums, counts = kf.oracle_fx(d)
    per = sums[0] // (1 << 16)
    assert sums[0] == per * (1 << 16) and sums[1] == -sums[0]
    T = (1 << 22) + 5
    assert (1 << 83) < per * T < 1 << 84                               # passes 2^83


@pytest.mark.parametrize("mode", ["mixed", "equal", "sparse"])
def test_score_keys(orc, mode):
    C = 1024
    d = kf.key_dims(C, mode)
    sums, counts = kf.oracle_fx(d)
    assert (sums, counts) == kf.key_targets(C, mode)
    sc = kf.scores_of(sums, counts)
    keys = [kf.score_key(s) for s in sc]
    if mode == "equal":
        assert len(set(keys)) == 1
        return
    assert any(np.isneginf(sc))
    ok = sc[~np.isneginf(sc)]
    order = np.argsort(-sc, kind="stable")
    assert list(order) == list(kf.sharding.topk_indices(sc, C))
    if mode == "sparse":
        assert np.isneginf(sc).sum() >= 3 * C // 4 and kf.straddling_k(sc) is not None
        return
    assert len(ok) > C // 2
    # within class j (c mod 17 == j < 14) distinct scores share exactly their top 7 - j % 7 bytes (and no more)
    for j in range(14):
        ks = sorted({keys[c] for c in range(j, C, 17)})
        assert len(ks) > 8
        shared = 7 - j % 7
        assert len({k >> (64 - 8 * shared) for k in ks}) == 1
        assert len({k >> (64 - 8 * shared - 8) for k in ks}) > 1
    assert len({k >> 56 for k in keys}) > 4                          # the top byte differs across classes
    k = kf.straddling_k(sc)
    o = kf.sharding.topk_indices(sc, C)
    assert sc[o[k - 1]] == sc[o[k]]
    assert kf.k_values(sc) == sorted({0, 1, k, C})


def test_host_out_edges():
    for kc in (lambda C: 1, lambda C: C):
        C = kf.host_out_edge(kc)
        assert kf.result_bytes(C, kc(C)) <= kf.HOST_OUT_MAX < kf.result_bytes(C + 1, kc(C + 1))
    assert kf.result_bytes(1, 1) % 16 == 0
    sizes = kf.k3_sizes()
    assert {1, 1024, 1025, 2048, 2049, 4096} <= set(sizes) and len(sizes) >= 13


@pytest.mark.parametrize("w", [None, np.array([0.3, 0.1, 0.05, 0.05, 0.1, 0.1, 0.1, 0.1, 0.1])])
def test_fx_model_is_the_oracle_on_shape_rows(orc, w):
    d = kf.shape_dims(3, 3000)
    assert kf.fx_model(d, w=w) == kf.oracle_fx(d, w=w)
    s = kf.short_dims(40, 7)
    assert kf.fx_model(s, w=w) == kf.oracle_fx(s, w=w)
    r_s, r_n = kf.fx_model(d, w=w, recip=True)
    e_s, e_n = kf.oracle_fx(d, w=w)
    assert r_n == e_n and all(abs(a - b) <= 3000 * 2 ** 10 for a, b in zip(r_s, e_s))    # recip: <= 1 ulp per evaluation
