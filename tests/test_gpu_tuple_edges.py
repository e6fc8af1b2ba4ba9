"""Form T at its edges on the H100 (-m gpu): k_tuple_values and K1t (csrc/apo_tuple.cu) on hand-built dictionaries and index
planes (tests/tuple_fixtures.py), resident (apo_score, source APO_SRC_TUPLES) and streamed from pageable and page-locked host
memory (apo_score_host_tuples).

Every case compares debug_partials (sums and counts) with the CPU reference with no tolerance, the scores bit for bit with
sharding.scores_from_partials of the reference integers, and the top-K with the oracle's.  Dictionary sizes sit around the
shared-memory head (hot = min(n + 1, 24576): the zero sentinel moves from shared memory to global), where th becomes
non-zero, at 2^20 + 3 and at 2^24 - 1; the planes put 8 different high bytes in every group of 8, boundary indices at fixed
positions, whole warps on one entry, reads that all miss the head, lanes on one bank pair; groups of 8 maximal entries
sit next to K1t's count field.  Refusals: indices == n_tuples and 0xFFFFFF in full and ragged tiles, entries at +-2.0, and
entries that name an empty or NaN slot of either codebook (also unreferenced: entries are checked, not evaluations), and
Form P evaluations that name such slots (k_unpack_p)."""
import importlib

import numpy as np
import pytest

import tuple_fixtures as tf
from test_gpu_candidates import eng_list, orc_rep

pytestmark = pytest.mark.gpu

sharding = importlib.import_module("senweaver-ide_b200.sharding")
BOOK, D2B = tf.codebook(), tf.d2book()
APO_E_ARG, APO_E_STATE = -1, -3
SHAPES = [(3, T) for T in tf.T_EDGES] + [(300, 8193)]     # (300, 8193): 600 tiles, candidates change inside a CTA's range


@pytest.fixture(scope="module")
def oc(orc):
    from oracle import candidates
    candidates.build()
    return candidates


def check(engine, orc, res, want, C):
    sums, counts = want
    assert engine.debug_partials(C) == (sums, counts)
    scores = sharding.scores_from_partials(sums, counts)
    assert res.scores.tobytes() == scores.tobytes()
    assert [int(x) for x in res.counts] == counts
    assert np.array_equal(res.topk, orc.topk(scores, len(res.topk)))


def pinned(apo, tl, th):
    ptl, pth = apo.host_empty(tl.shape, np.uint16), apo.host_empty(th.shape, np.uint8)
    ptl[:], pth[:] = tl, th
    return ptl, pth


def score_all(engine, apo, orc, idx, tb, want, page_locked=True, recip=False):
    """streamed (pageable, then page-locked) and resident: all equal `want`"""
    C = idx.shape[0]
    K = min(C, 3)
    tl, th = tf.planes(idx)
    check(engine, orc, engine.score_host_tuples(tl, th, tb, BOOK, D2B, K, recip=recip), want, C)
    if page_locked:
        check(engine, orc, engine.score_host_tuples(*pinned(apo, tl, th), tb, BOOK, D2B, K, recip=recip), want, C)
    engine.tuples_upload(tl, th, tb, BOOK, D2B)
    check(engine, orc, engine.score(C, K, source=apo.SRC_TUPLES, recip=recip), want, C)


def refused(apo, call, code=APO_E_ARG):
    with pytest.raises(apo.ApoError) as ei:
        call()
    assert ei.value.code == code


@pytest.mark.parametrize("n", tf.SIZES[:-1])
def test_dictionary_sizes_and_index_planes(engine, orc, apo, n):
    tb = tf.dictionary(n)
    fx, counted = tf.entry_fx(tb, BOOK, D2B)
    for name, build in tf.PLANES.items():
        for k, (C, T) in enumerate(SHAPES):
            idx = build(n, C, T, seed=k)
            score_all(engine, apo, orc, idx, tb, tf.expected(idx, fx, counted), page_locked=k == 5)


@pytest.mark.parametrize("n", [24577, 65537, (1 << 20) + 3])
def test_maximal_entries_next_to_the_count_field(engine, orc, apo, n):
    tb = tf.dictionary(n)
    try:
        for w in (None, tf.ZERO_W):
            if w is not None:
                engine.set_weights(w)
            fx, counted = tf.entry_fx(tb, BOOK, D2B, w=w)
            for C, T in ((3, 16385), (5, 8193), (2, 7), (300, 8193)):
                idx = tf.max_groups(n, C, T)
                score_all(engine, apo, orc, idx, tb, tf.expected(idx, fx, counted), page_locked=C == 5)
    finally:
        engine.set_weights(orc.weights())


def test_windows_start_on_groups_and_end_anywhere(engine, orc, apo):
    n, C, T = 65537, 5, 40_003
    tb = tf.dictionary(n)
    fx, counted = tf.entry_fx(tb, BOOK, D2B)
    idx = np.concatenate([tf.hi_byte_groups(n, 2, T), tf.boundary(n, 2, T), tf.max_groups(n, 1, T)])
    engine.tuples_upload(*tf.planes(idx), tb, BOOK, D2B)
    for first, count in ((8, 8191), (0, 8193), (8192, 8193), (16, 1), (8184, 16385), (24576, 7), (40_000, 3), (32_768, 7235)):
        r = engine.score(C, 2, source=apo.SRC_TUPLES, first=first, count=count)
        check(engine, orc, r, tf.expected(idx[:, first:first + count], fx, counted), C)


def test_streamed_windows_cut_rows_with_a_ragged_last_chunk(engine, orc, apo):
    n, C, T = (1 << 20) + 3, 4096, 40_000
    assert tf.stream_chunks(C, T) == 3
    tb = tf.dictionary(n)
    fx, counted = tf.entry_fx(tb, BOOK, D2B)
    idx = tf.hi_byte_groups(n, C, T)
    idx[::7] = tf.max_groups(n, len(idx[::7]), T)
    score_all(engine, apo, orc, idx, tb, tf.expected(idx, fx, counted))


def test_largest_dictionary(engine, orc, apo):
    n = tf.TUPLES_MAX
    tb = tf.dictionary(n)
    fx, counted = tf.entry_fx(tb, BOOK, D2B)
    idx = np.concatenate([tf.uniform(n, 24, 40_003), tf.hi_byte_groups(n, 24, 40_003), tf.max_groups(n, 8, 40_003),
                          tf.reversed_freq(n, 8, 40_003), tf.boundary(n, 8, 40_003)])
    assert len(np.unique(idx >> 16)) == 256
    score_all(engine, apo, orc, idx, tb, tf.expected(idx, fx, counted))


@pytest.mark.parametrize("weights", ["default", "recip", "custom", "zero", "ones_significand"])
def test_weights_and_division(engine, orc, apo, weights):
    n, C, T = 24577, 7, 20_003
    tb = tf.dictionary(n)
    idx = np.concatenate([tf.boundary(n, 3, T), tf.max_groups(n, 2, T), tf.warp_uniform(n, 2, T)])
    w = {"default": None, "recip": None, "custom": np.array([0.3, 0.05, 0.1, 0.05, 0.1, 0.1, 0.1, 0.1, 0.1]),
         "zero": tf.ZERO_W, "ones_significand": tf.ONES_W}[weights]
    try:
        if w is not None:
            engine.set_weights(w)
        if weights == "recip":
            # Form T's integers are Form D's recip integers on the decoded tensor
            engine.dims_upload(tf.rows_of(idx, tb, BOOK, D2B))
            rd = engine.score(C, 3, recip=True)
            want = engine.debug_partials(C)
            score_all(engine, apo, orc, idx, tb, want, recip=True)
            assert np.array_equal(rd.scores, sharding.scores_from_partials(*want))
        else:
            fx, counted = tf.entry_fx(tb, BOOK, D2B, w=w)
            want = tf.expected(idx, fx, counted)
            if weights == "zero":
                assert min(want[1]) < T                  # null entries are met and not counted
            score_all(engine, apo, orc, idx, tb, want)
    finally:
        engine.set_weights(orc.weights())


def test_sessions_sum_windows_and_keep_a_refusal(engine, orc, apo):
    n, C, T = 65537, 4, 30_001
    tb = tf.dictionary(n)
    fx, counted = tf.entry_fx(tb, BOOK, D2B)
    idx = np.concatenate([tf.hi_byte_groups(n, 2, T), tf.max_groups(n, 2, T)])
    tl, th = tf.planes(idx)
    engine.tuples_upload(tl, th, tb, BOOK, D2B)
    want = tf.expected(idx, fx, counted)
    engine.score_begin(C)
    engine.score_accumulate(0, source=apo.SRC_TUPLES, first=16_384)               # the second window first
    engine.score_accumulate(0, source=apo.SRC_TUPLES, first=0, count=16_384)
    check(engine, orc, engine.score_finish(C, 2), want, C)
    # an index == n_tuples in the FIRST window: the flag survives the clean second window and fails the finish
    bad_l, bad_h = tl.copy(), th.copy()
    bad_l[1, 77], bad_h[1, 77] = n & 0xFFFF, n >> 16
    engine.tuples_upload(bad_l, bad_h, tb, BOOK, D2B)
    engine.score_begin(C)
    engine.score_accumulate(0, source=apo.SRC_TUPLES, first=0, count=8192)
    engine.score_accumulate(0, source=apo.SRC_TUPLES, first=8192)
    refused(apo, lambda: engine.score_finish(C, 2))
    r = engine.score(C, 2, source=apo.SRC_TUPLES, first=8192)                    # the next call is exact
    check(engine, orc, r, tf.expected(idx[:, 8192:], fx, counted), C)


@pytest.mark.parametrize("where", ["full_tile", "ragged_tail"])
@pytest.mark.parametrize("bad_index", ["n_tuples", "0xFFFFFF"])
def test_index_outside_the_dictionary_is_refused(engine, orc, apo, where, bad_index):
    n, C, T = 65537, 3, 2 * 8192 + 9
    tb = tf.dictionary(n)
    fx, counted = tf.entry_fx(tb, BOOK, D2B)
    idx = tf.hi_byte_groups(n, C, T)
    want = tf.expected(idx, fx, counted)
    bad = idx.copy()
    bad[1, 8192 + 101 if where == "full_tile" else T - 2] = n if bad_index == "n_tuples" else 0xFFFFFF
    tl, th = tf.planes(bad)
    refused(apo, lambda: engine.score_host_tuples(tl, th, tb, BOOK, D2B, 1))
    check(engine, orc, engine.score_host_tuples(*tf.planes(idx), tb, BOOK, D2B, 2), want, C)
    engine.tuples_upload(tl, th, tb, BOOK, D2B)
    refused(apo, lambda: engine.score(C, 1, source=apo.SRC_TUPLES, candidates=True))
    refused(apo, lambda: engine.candidate_reports(0, C), APO_E_STATE)
    engine.tuples_upload(*tf.planes(idx), tb, BOOK, D2B)
    check(engine, orc, engine.score(C, 2, source=apo.SRC_TUPLES), want, C)


@pytest.mark.parametrize("referenced", [True, False])
@pytest.mark.parametrize("name", tf.BAD)
def test_unrepresentable_entries_are_refused(engine, orc, apo, oc, name, referenced):
    """+-2.0, an empty or NaN tool_success_rate slot, an empty or NaN coded slot: APO_E_ARG whether or not an evaluation
    names the entry (k_tuple_values checks entries), resident and streamed; the handle stays usable and exact"""
    n, C, T = 24577, 3, 8193
    where = n - 7                                                  # in the tail of the dictionary
    tb = tf.dictionary(n, {**tf.default_places(n), name: where})
    clean = tf.dictionary(n)
    fx, counted = tf.entry_fx(clean, BOOK, D2B)
    idx = tf.boundary(n, C, T)
    idx[idx == where] = 0
    if referenced:
        idx[2, 4096:4104] = where
    tl, th = tf.planes(idx)
    refused(apo, lambda: engine.score_host_tuples(tl, th, tb, BOOK, D2B, 1, candidates=True))
    refused(apo, lambda: engine.candidate_reports(0, C), APO_E_STATE)
    engine.tuples_upload(tl, th, tb, BOOK, D2B)
    refused(apo, lambda: engine.score(C, 1, source=apo.SRC_TUPLES))
    refused(apo, lambda: engine.score(C, 1, source=apo.SRC_TUPLES, candidates=True))
    refused(apo, lambda: engine.candidate_reports(0, C), APO_E_STATE)
    clean_idx = idx.copy()
    clean_idx[clean_idx == where] = 1
    score_all(engine, apo, orc, clean_idx, clean, tf.expected(clean_idx, fx, counted), page_locked=False)


@pytest.mark.parametrize("name", ["code_empty", "code_nan", "d2_empty", "d2_nan"])
def test_packed_evaluations_naming_empty_slots_are_refused(engine, orc, apo, name):
    """Form P streamed (k_unpack_p -> K1q) refuses an evaluation that names an empty or NaN slot of either codebook; the
    same planes without it give the oracle's integers"""
    n, C, T = 64, 4, 2 * 8192 + 5
    places = {**tf.default_places(n), name: 40}
    tb = tf.dictionary(n, places)
    fx, counted = tf.entry_fx(tb, BOOK, D2B)
    idx = tf.uniform(n, C, T)
    idx[idx == 40] = 0
    want = tf.expected(idx, fx, counted)
    pc, pd = tb[0][idx], tb[1][idx]
    check(engine, orc, engine.score_host_packed(pc, pd, BOOK, D2B, 2), want, C)
    pc[3, T - 1], pd[3, T - 1] = tb[0][40], tb[1][40]
    refused(apo, lambda: engine.score_host_packed(pc, pd, BOOK, D2B, 1))
    refused(apo, lambda: engine.score_host_packed(pc, pd, BOOK, D2B, 1, candidates=True))
    refused(apo, lambda: engine.candidate_reports(0, C), APO_E_STATE)
    pc[3, T - 1], pd[3, T - 1] = tb[0][idx[3, T - 1]], tb[1][idx[3, T - 1]]
    check(engine, orc, engine.score_host_packed(pc, pd, BOOK, D2B, 2), want, C)


@pytest.mark.parametrize("n", [24576, 65537])
def test_breakdown_equals_the_oracle_on_the_decoded_rows(engine, orc, apo, oc, n):
    C, T = 5, 16_385
    tb = tf.dictionary(n)
    idx = np.concatenate([tf.max_groups(n, 2, T), tf.hi_byte_groups(n, 1, T), tf.boundary(n, 1, T), tf.warp_uniform(n, 1, T)])
    ref = [orc_rep(d) for d in oc.cand_dims(tf.rows_of(idx, tb, BOOK, D2B))]
    tl, th = tf.planes(idx)
    assert eng_list(engine.score_host_tuples(tl, th, tb, BOOK, D2B, 2, candidates=True).candidates) == ref
    engine.tuples_upload(tl, th, tb, BOOK, D2B)
    assert eng_list(engine.score(C, 2, source=apo.SRC_TUPLES, candidates=True).candidates) == ref
