"""The long-session legs without a GPU (tests/long_session_fixtures.py): every leg of tests/test_gpu_long_sessions.py crosses a
wrap of the words as the engine kept them before, and none under the words and the limb guard it keeps now, at the SM counts of
an H100 SXM (132) and PCIe (114); the restatements agree with exact sums on small cases."""
import numpy as np
import pytest

import group_fixtures as gf
import long_session_fixtures as lf
import spread_fixtures as sf
import tuple_fixtures as tf

SMS = (132, 114)
MAXV = float(tf.MAXV)


def test_restatements_agree_on_small_cases():
    rng = np.random.default_rng(7)
    for _ in range(200):
        xs = [int(v) for v in rng.integers(-(1 << 62), 1 << 62, 40)]
        terms = {}
        for x in xs:
            terms[x] = terms.get(x, 0) + 1
        assert not lf.group_wraps(terms)
        assert lf.parent_group_sum(terms) == lf.fixed_group_sum(terms) == sum(xs)
        lanes = [int(v) for v in rng.integers(-(1 << 40), 1 << 40, 32)]
        limbs = lf.flush_limbs(lanes)
        assert lf.exact_limbs(1, limbs) == sum(lanes)
        assert lf.parent_limbs_read(1000, limbs) == 1000 * sum(lanes)
        assert max(limbs[0], limbs[1]) <= lf.FLUSH_ADD_MAX


def test_parent_limbs_wrap_where_the_issue_counts():
    limbs = lf.LIMBS_ONE
    assert limbs[1] == 32 * (2 ** 32 - 1)
    F = lf.l1_wrap_flushes(limbs)
    assert F == 67_108_865
    assert lf.parent_limbs_read(F - 1, limbs) == lf.exact_limbs(F - 1, limbs) == -(F - 1) * 32
    # l1 and l0 (whose lane halves are 2^32 - 1 as well) both read negative: 2^96 + 2^64 units off
    assert lf.parent_limbs_read(F, limbs) == lf.exact_limbs(F, limbs) - (1 << 96) - (1 << 64)


def _leg_a_fx():
    return {0: -int(MAXV * 2 ** 52), 1: int(MAXV * 2 ** 52), 2: None}


def test_leg_a_groups_wrap_only_at_32():
    fx = _leg_a_fx()
    fx[2] = fx[0] + 12345                           # any term of the same sign: one evaluation does not move a wrap
    assert lf.A_N0 + lf.A_N1 + lf.A_N2 == lf.A_T and lf.A_N0 == lf.A_N1
    for k in lf.A_K:
        t = lf.leg_a_group_terms(fx, k)
        want = (k == 32, k == 32, False)
        assert tuple(lf.group_wraps(g) for g in t) == want, k
        for g, w in zip(t, want):
            assert (lf.parent_group_sum(g) != lf.fixed_group_sum(g)) == w
            assert lf.fixed_group_sum(g) == sum(x * n for x, n in g.items())
    # group 0 at 32 passes word 1's wrap (~(2^32 + 2^21) negative terms), group 1 word 0's (8/7 2^32 positive terms)
    assert 32 * lf.A_N0 > (2 ** 64) // (2 ** 32 - 2 ** 21) and 32 * lf.A_N1 * 3 * 2 ** 30 >= 2 ** 64
    assert 8 * lf.A_N0 * (2 ** 32 - 2 ** 21) < 2 ** 64


def test_leg_a_planes_and_labels():
    tl, th = lf.leg_a_planes()
    labels = lf.leg_a_labels()
    assert tl.shape == (1, lf.A_T) and not th.any()
    for g, counts in enumerate(lf.leg_a_counts()):
        sel = tl[0][labels == g]
        assert {int(e): int((sel == e).sum()) for e in np.unique(sel)} == counts
    pc, pd = lf.leg_a_dictionary()
    rows = tf.decode((pc, pd), tf.codebook(), tf.d2book())
    assert rows[0, 8] == -tf.MAXV and rows[1, 8] == tf.MAXV and rows[2, 0] == -1.0 and rows[2, 8] == -tf.MAXV
    assert np.isnan(rows[:2, :8]).all()


@pytest.mark.parametrize("sm", SMS)
def test_leg_b_crosses_the_parent_wrap_and_not_the_guarded_one(sm):
    n = lf.leg_b_accumulates(sm)
    F = lf.l1_wrap_flushes(lf.LIMBS_ONE)
    fewest = lf.PASS_MIN_WARPS_PER_SM * sm
    assert min(lf.K1_WARPS_PER_SM, lf.K1T_WARPS_PER_SM, lf.PASS_MIN_WARPS_PER_SM) == lf.PASS_MIN_WARPS_PER_SM
    assert n * fewest >= F * 1.1 > (n - 1) * fewest           # every launch shape of the leg crosses, with the margin
    if sm == 132:
        assert 69_000 < n < 71_000
    first = lf.leg_b_first_checkpoint(sm)
    assert first * lf.MAX_WARPS_PER_SM * sm < F                # before any launch shape could cross
    assert lf.parent_limbs_read(n * fewest, lf.LIMBS_ONE) != lf.exact_limbs(n * fewest, lf.LIMBS_ONE)
    carries, worst = lf.limb_guard([lf.B_T] * n, sm)
    assert carries >= 8 and worst <= lf.LIMB_FLUSH_MAX
    assert lf.limb_words_max(lf.LIMB_FLUSH_MAX) < 2 ** 63
    assert lf.limb_guard([lf.B_T] * first, sm)[0] == 0         # the first checkpoint is reached before any carry
    # the G = 1 group words under the old arithmetic: n B_T terms at x = -1 pass word 1's 2^64
    terms = {-1: n * lf.B_T}
    assert lf.group_wraps(terms) and lf.parent_group_sum(terms) != lf.fixed_group_sum(terms) == -n * lf.B_T
    m = sf.fields(n * lf.B_T, -n * lf.B_T, n * lf.B_T)
    assert m["M"] == 0 and m["mean"] == -2.0 ** -52
    assert gf.score_of(n * lf.B_T, 0, 0, n * lf.B_T, -n * lf.B_T)["avgReward"] == -2.0 ** -52


@pytest.mark.parametrize("sm", SMS)
def test_no_guarded_launch_sequence_passes_2_63(sm):
    """the guard over windows of every size, from one evaluation to 2^36 (one launch reads a window held on the device: 80 GB
    hold fewer than 2^36 evaluations of any layout)"""
    for count in (1, lf.B_T, lf.A_T, lf.C_T_WIDE, 1 << 36):
        carries, worst = lf.limb_guard([count] * 5000, sm)
        assert worst <= lf.LIMB_FLUSH_MAX and lf.limb_words_max(worst) < 2 ** 63
    assert lf.limb_guard([1] * 100, sm) == (0, 100 * lf.limb_flush_bound(1, sm))   # a short session carries nothing


def test_leg_c_passes_the_parent_group_words():
    assert lf.leg_c_group_terms_wrap(lf.C_T_WIDE)             # 2^34 random terms per candidate: word 0 passes 2^64
    assert not lf.leg_c_group_terms_wrap(lf.C_T_WIDE // 4)
