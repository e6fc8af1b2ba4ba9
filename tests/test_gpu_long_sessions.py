"""Long scoring sessions on the H100, against exact integers with no tolerance (tests/long_session_fixtures.py):

- A: one resident Form T row of 2^29 + 33 evaluations in three groups, accumulated 32 times, so that groups 0 and 1 each
  take 1.5 * 2^32 terms at -(2 - 2^-23) and +(2 - 2^-23): scores, partials, breakdown, every group field, every spread
  field by its bytes and both extremes lists after 8 and 32 accumulates, in closed form.
- B: constant rows at fr = -2^-52 accumulated ~70 000 times (leg_b_accumulates), past the point where the candidate
  partials', the breakdown's and the group words' 32-bit limbs would pass 2^63 without the limb carry, through Form D (K1),
  the Form T copy (K1t) and resident Form T, finished before and after.
- C: generator rows on every route scored once, then accumulated 128 times in one session: every integer of every report
  128 times the single call's, every ratio unchanged, the spread rebuilt from the scaled integers, the extremes lists the
  single call's first key 32 times.  Each candidate takes 2^34 random terms."""
import math
import struct

import numpy as np
import pytest

import exact_report as xr
import oracle
import group_fixtures as gf
import long_session_fixtures as lf
import spread_fixtures as sf
import tuple_fixtures as tf
from extremes_fixtures import rows

pytestmark = pytest.mark.gpu
FLAGS4 = dict(candidates=True, extremes=True, groups=True, spread=True)


def bits(v) -> bytes:
    return struct.pack("<d", float(v))


def spread_tuple(s) -> tuple:
    return (int(s.n), int(s.sumLo), int(s.sumHi), int(s.sumSq[0]), int(s.sumSq[1]), int(s.sumSq[2]), bits(s.mean), bits(s.rewardSumSq),
            bits(s.variance), bits(s.stdDev), bits(s.stdErr))


def spread_ref(m: dict) -> tuple:
    return tuple(bits(m[f]) if isinstance(m[f], float) else int(m[f]) for f in sf.FIELDS)


def check_group(got, m: dict, where):
    assert (int(got.total), int(got.good), int(got.bad), int(got.withReward)) == (m["total"], m["good"], m["bad"], m["withReward"]), where
    assert (bits(got.goodRate), bits(got.rewardSum), bits(got.avgReward)) == (bits(m["goodRate"]), bits(m["rewardSum"]), bits(m["avgReward"])), where


def fx_double(s: int) -> float:
    return float(s) / float(lf.FX)                # one rounding of the integer, exact scaling


# ------------------------------------------------------------------------------------------------ A
def test_a_group_words_past_2_32_terms(engine, orc, apo):
    pc, pd = lf.leg_a_dictionary()
    book, d2b = tf.codebook(), tf.d2book()
    fx, counted = tf.entry_fx((pc, pd), book, d2b, sf.w_one())
    assert counted.all()
    tl, th = lf.leg_a_planes()
    labels = lf.leg_a_labels()
    lo_e, hi_e = int(np.argmin(fx)), int(np.argmax(fx))
    idx = tl[0]
    first_lo = np.flatnonzero(idx == lo_e)[:32]
    first_hi = np.flatnonzero(idx == hi_e)[:32]
    d8 = {e: int(round(float(tf.decode((pc, pd), book, d2b)[e, 8]) * lf.FX)) for e in range(3)}
    try:
        engine.set_weights(sf.w_one())
        engine.tuples_upload(tl, th, (pc, pd), book, d2b)
        engine.record_groups_upload(labels, lf.A_G)
        del tl, th, labels
        engine.score_begin(1)
        for k in range(1, max(lf.A_K) + 1):
            engine.score_accumulate(0, source=apo.SRC_TUPLES, **FLAGS4)
            if k not in lf.A_K:
                continue
            res = engine.score_finish(1, 1, **FLAGS4)
            counts = [{e: k * n for e, n in g.items()} for g in lf.leg_a_counts()]
            n = k * lf.A_T
            S = sum(int(fx[e]) * m for g in counts for e, m in g.items())
            S2 = sum(int(fx[e]) ** 2 * m for g in counts for e, m in g.items())
            assert engine.debug_partials(1) == ([S], [n]), k
            assert int(res.counts[0]) == n and bits(res.scores[0]) == bits(math.ldexp(float(S), -52) / float(n)), k
            for g, (cnt, terms) in enumerate(zip(counts, lf.leg_a_group_terms(fx, k))):
                tot = sum(cnt.values())
                check_group(res.groups[0][g], gf.score_of(tot, 0, k if g == 0 else 0, tot, lf.fixed_group_sum(terms)), (k, g))
            assert spread_tuple(res.spread[0]) == spread_ref(sf.fields(n, S, S2)), k
            r = res.candidates[0]
            assert (int(r.total), int(r.good), int(r.bad), int(r.none), int(r.withReward)) == (n, 0, k, n - k, n), k
            assert bits(r.rewardSum) == bits(fx_double(S)), k
            s8 = sum(d8[e] * m for g in counts for e, m in g.items())
            assert (bits(r.dim[0].sum), int(r.dim[0].count)) == (bits(fx_double(-k * lf.FX)), k), k
            assert (bits(r.dim[8].sum), int(r.dim[8].count)) == (bits(fx_double(s8)), n), k
            assert all(int(r.dim[i].count) == 0 for i in range(1, 8)), k
            x = res.extremes[0]
            per = -(-32 // k)
            want_lo = [int(p) for p in first_lo[:per] for _ in range(k)][:32]
            want_hi = [int(p) for p in first_hi[:per] for _ in range(k)][:32]
            assert int(x.n) == 32 and list(x.lowest) == want_lo and list(x.highest) == want_hi, k
            assert {bits(v) for v in x.lowestReward} == {bits(fx_double(int(fx[lo_e])))}, k
            assert {bits(v) for v in x.highestReward} == {bits(fx_double(int(fx[hi_e])))}, k
    finally:
        engine.record_groups_upload(np.zeros(0, np.uint8), 0)
        engine.set_weights(oracle.weights())


# ------------------------------------------------------------------------------------------------ B
B_ROUTES = {"k1": (0x10, False), "t_copy_k1t": (0x40 | 0x80 | 0x100, False), "tuples": (0, True)}


@pytest.mark.parametrize("route", list(B_ROUTES))
def test_b_limbs_past_2_26_flushes(engine, apo, route):
    import torch
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    checkpoints = lf.leg_b_checkpoints(sm)
    tune, tuples = B_ROUTES[route]
    flags = dict(FLAGS4) if tuples else dict(candidates=True, groups=True, spread=True)
    src = apo.SRC_TUPLES if tuples else apo.SRC_DIMS
    d = rows(lf.B_T, d1=np.float32(-2.0 ** -52))[None]
    try:
        engine.set_weights(sf.w_one())
        engine.set_tuning(tune)
        engine.dims_upload(d)
        if tuples:
            engine.dims_tuples()
        engine.record_groups_upload(np.zeros(lf.B_T, np.uint8), 1)
        engine.score_begin(1)
        done = 0
        for k in checkpoints:
            while done < k:
                engine.score_accumulate(0, source=src, **flags)
                done += 1
            res = engine.score_finish(1, 1, **flags)
            n = k * lf.B_T
            where = (route, k)
            assert engine.debug_partials(1) == ([-n], [n]), where
            assert bits(res.scores[0]) == bits(-2.0 ** -52) and int(res.counts[0]) == n, where
            r = res.candidates[0]
            assert (int(r.total), int(r.withReward), bits(r.rewardSum)) == (n, n, bits(fx_double(-n))), where
            assert (bits(r.dim[1].sum), int(r.dim[1].count)) == (bits(fx_double(-n)), n), where
            check_group(res.groups[0][0], gf.score_of(n, 0, 0, n, -n), where)
            assert spread_tuple(res.spread[0]) == spread_ref(sf.fields(n, -n, n)), where
            if tuples:
                x = res.extremes[0]
                assert int(x.n) == 32 and list(x.lowest) == [0] * 32 and list(x.highest) == [0] * 32, where
    finally:
        engine.set_tuning(0)
        engine.record_groups_upload(np.zeros(0, np.uint8), 0)
        engine.set_weights(oracle.weights())


# ------------------------------------------------------------------------------------------------ C
def _scaled_struct(a, b, ints, sums, same, where):
    s = lf.C_SCALE
    for f in ints:
        assert int(getattr(b, f)) == s * int(getattr(a, f)), (where, f)
    for f in sums:
        assert bits(getattr(b, f)) == bits(s * getattr(a, f)), (where, f)
    for f in same:
        va, vb = getattr(a, f), getattr(b, f)
        assert (bits(vb) == bits(va)) if isinstance(va, float) else vb == va, (where, f)


def first_three(ex) -> list:
    """the first-three slots of a session that read the same window C_SCALE times: the single call's first position in each
    slot (every position comes back once per accumulate), -1 when there is none"""
    return [int(ex[0])] * 3


def _dims(a, b, where):
    for i in range(9):
        _scaled_struct(a.dim[i], b.dim[i], ("count",), ("sum",), ("avg", "low_flag", "low_severity", "sugg_flag", "sugg_priority"), (where, i))


def check_scaled(one, ses, engine, C, G, where):
    s = lf.C_SCALE
    assert bytes(ses.scores) == bytes(one.scores) and list(ses.counts) == [s * int(v) for v in one.counts], where
    for c in range(C):
        a, b = one.candidates[c], ses.candidates[c]
        _scaled_struct(a, b, ("total", "good", "bad", "none", "withReward"), ("rewardSum",), ("goodRate", "avgReward"), (where, c))
        assert list(b.badExamples) == first_three(a.badExamples), (where, c)
        _dims(a, b, (where, c))
        for g in range(G):
            _scaled_struct(one.groups[c][g], ses.groups[c][g], ("total", "good", "bad", "withReward"), ("rewardSum",),
                           ("goodRate", "avgReward"), (where, c, g))
        sp = one.spread[c]
        assert spread_tuple(ses.spread[c]) == spread_ref(sf.fields(s * int(sp.n), s * sp.sum, s * sp.sum_sq)), (where, c)
        xa, xb = one.extremes[c], ses.extremes[c]
        assert int(xb.n) == int(xa.n) == 32, (where, c)
        for lst, rew in (("lowest", "lowestReward"), ("highest", "highestReward")):
            assert list(getattr(xb, lst)) == [getattr(xa, lst)[0]] * 32, (where, c, lst)
            assert {bits(v) for v in getattr(xb, rew)} == {bits(getattr(xa, rew)[0])}, (where, c, rew)
    sums, counts = engine.debug_partials(C)
    assert counts == [int(v) for v in ses.counts], where
    return sums


def check_scaled_corpus(a, b, where):
    s = lf.C_SCALE
    _scaled_struct(a, b, ("total", "good", "bad", "none", "withReward", "toolCalls", "toolSucc", "toolFail"), ("rewardSum",),
                   ("goodRate", "avgReward", "toolSuccessRate"), where)
    assert [[s * int(v) for v in m] for m in a.byMode] == [[int(v) for v in m] for m in b.byMode], where
    assert bytes(a.byModeGoodRate) == bytes(b.byModeGoodRate), where
    _dims(a, b, where)
    for p in range(xr.NPAT):
        pa, pb = a.pat[p], b.pat[p]
        assert int(pb.count) == s * int(pa.count) and list(pb.examples) == first_three(pa.examples), (where, p)
        if pa.flag:                                  # a flagged pattern stays flagged; its severity follows the scaled count
            assert pb.flag and pb.severity == xr.pattern_severity(p, s * int(pa.count)), (where, p)
        elif int(pa.count) == 0:
            assert not pb.flag, (where, p)


def _single_and_session(engine, C, source, flags, labels_G):
    one = engine.score(C, 1, source=source, **flags)
    one_sums, one_counts = engine.debug_partials(C)
    engine.score_begin(C)
    for _ in range(lf.C_SCALE):
        engine.score_accumulate(0, source=source, **flags)
    ses = engine.score_finish(C, 1, **flags)
    sums = check_scaled(one, ses, engine, C, labels_G, flags)
    assert sums == [lf.C_SCALE * v for v in one_sums] and one_counts == [int(v) for v in one.counts]
    return one, ses


C_ROUTES = {"k1": 0x10, "w_copy": 0x20, "t_copy": 0x40, "default": 0}


def test_c_random_rows_every_route_scaled(orc, apo):
    """C = 2 rows of 2^27 + 9 generator evaluations (9.7 GB as Form D) on an engine of its own, closed at the end; G = 2
    (group 1: every 1024th record) so that group 0 takes ~2^34 random terms per candidate"""
    C, T, G = 2, lf.C_T_WIDE, 2
    labels = (np.arange(T) % 1024 == 1023).astype(np.uint8)
    e = apo.Engine(0)
    try:
        e.record_groups_upload(labels, G)
        for route, tune in C_ROUTES.items():
            e.set_tuning(tune)
            e.dims_generate(0x5EED9001, 0, C, 0, T, 300)
            _single_and_session(e, C, apo.SRC_DIMS, dict(FLAGS4, groups=True), G)
        e.set_tuning(0)
        e.dims_tuples()
        _single_and_session(e, C, apo.SRC_TUPLES, dict(FLAGS4), G)           # resident Form T built on the device
        e.dims_generate_compact(0x5EED9001, 0, C, 0, T, 300)
        _single_and_session(e, C, apo.SRC_DIMS, dict(FLAGS4), G)             # resident Form Q
        e.rollouts16_generate(0x5EED9002, 0, C, 0, T, 300)
        flags = dict(FLAGS4, candidate_corpus=True)
        one, ses = _single_and_session(e, C, apo.SRC_ROLLOUTS, flags, G)      # R16
        for c in range(C):
            check_scaled_corpus(one.candidate_corpus[c], ses.candidate_corpus[c], ("r16", c))
    finally:
        e.close()
