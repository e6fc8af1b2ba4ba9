"""The corpus builders of corpus_fixtures.py mean what they claim: on small instances the CPU oracle's report (oracle.report)
and breakdown (oracle.candidates) give exactly the designed counts and examples, and the closed form of a saturating corpus."""
import math

import numpy as np
import pytest

import corpus_fixtures as cf


@pytest.fixture(scope="module")
def oc(orc):
    from oracle import candidates
    candidates.build()
    return candidates


def check_against_closed_form(ref, want):
    """the oracle sums in sequential binary64: integers exactly, sums and averages to 1e-12"""
    assert (ref.total, ref.good, ref.bad, ref.none, ref.withReward) == (want["total"], 0, want["bad"], 0, want["withReward"])
    for m in range(5):
        assert list(ref.byMode[m]) == want["byMode"][m]
    assert math.isclose(ref.rewardSum, want["rewardSum"], rel_tol=1e-12, abs_tol=1e-12)
    for i, w in enumerate(want["dim"]):
        assert ref.dim[i].count == w["count"], i
        assert math.isclose(ref.dim[i].sum, w["sum"], rel_tol=1e-12, abs_tol=1e-12), i
        assert (ref.dim[i].low_flag, ref.dim[i].sugg_flag) == (w["low_flag"], w["sugg_flag"]), i
    for p, w in enumerate(want["pat"]):
        assert (ref.pat[p].count, ref.pat[p].flag, list(ref.pat[p].examples)) == (w["count"], w["flag"], w["examples"]), p
    assert (ref.toolCalls, ref.toolSucc, ref.toolFail) == (want["toolCalls"], want["toolSucc"], want["toolFail"])


@pytest.mark.parametrize("preds,mode", [((0, 2, 4), 1), ((1, 3, 5), 2), ((), 2), (tuple(range(6)), 4)])
def test_saturating_corpus_has_its_closed_form(orc, apo, preds, mode):
    T, base = 1000, (1 << 40) + 8
    recs = cf.saturating(T, preds, mode)
    want = cf.closed_form(T, preds, mode, idx_base=base)
    check_against_closed_form(orc.report(recs, idx_base=base), want)
    # every packed counter sees one category: a single dimension value per dimension, every dimension present
    d, m = orc.reward_dims(recs[:1])
    assert m == 0x1FF and all(w["count"] == T for w in want["dim"])
    if mode == 2:                                    # the agent thresholds: d6 of llmCalls <= 3 is 1, normal mode's is lower
        assert d[6] == 1.0 and orc.reward_dims(cf.hit_record(preds, 1))[0][6] < 1.0
    # Form R16 of the same records: the numpy packer is the engine's, and the report does not change
    p16 = cf.saturating(T, preds, mode, row=16)
    assert p16.tobytes() == apo.pack16(recs).tobytes()
    check_against_closed_form(orc.report(orc.unpack16(p16), idx_base=base), want)


def test_saturating_corpus_tiny_t_pads_examples(orc):
    want = cf.closed_form(2, (0, 1), 1, idx_base=5)
    assert want["pat"][0]["examples"] == [5, 6, -1] and want["pat"][0]["flag"] == 1
    check_against_closed_form(orc.report(cf.saturating(2, (0, 1)), idx_base=5), want)


@pytest.mark.parametrize("T,shift,base", [(20_000, 0, 0), (140_000, 37, (1 << 40) + 8), (300_001, 1000, 12)])
def test_planted_corpus_has_the_designed_patterns(orc, T, shift, base):
    recs, plan, want = cf.planted(T, shift=shift, idx_base=base)
    ref = orc.report(recs, idx_base=base)
    cf.check_designed(ref, want)
    for p in range(6):
        assert plan[p][0] > T // 6, p                                       # every earliest hit lies past the first warp's share
    assert ref.good > 0 and ref.none > 0 and ref.bad > len(set().union(*plan.values()))     # background 'bad' records hit nothing
    # the scenarios are what they say
    assert min(plan[0]) >= T - 2048 - shift - 1
    assert plan[1][0] % 32 == 31 and plan[1][-1] == T - 1
    assert all(q - 1 in plan[2] or q + 1 in plan[2] for q in plan[2])
    assert len({q // 32 for q in plan[3][1:]}) == 1 and len(plan[3]) > 4
    assert plan[4][-600:] == list(range(T - 600, T))
    # the same rows as Form R16
    p16 = cf.table(16)[cf.background_index(T)]
    assert p16.shape == (T,)
    recs16, _, want16 = cf.planted(T, shift=shift, row=16, idx_base=base)
    cf.check_designed(orc.report(orc.unpack16(recs16), idx_base=base), want16)


def test_planted_extra_positions_and_rotated_kinds(orc):
    T = 50_000
    recs, plan, want = cf.planted(T, kinds=(5, 4, 3, 2, 1, 0), extra={5: [100, 2047, 2048]})
    assert plan[5][:3] == [100, 2047, 2048]
    cf.check_designed(orc.report(recs), want)


def test_planted_rows_breakdown_and_sparse_bad_dims(orc, oc):
    C, T = 6, 30_000
    rows = np.stack([cf.planted(T, kinds=[(p + c) % 6 for p in range(6)], shift=64 * c)[0] for c in range(C)])
    for c, r in enumerate(oc.cand_records(rows, idx_base=7)):
        ref = orc.report(rows[c], idx_base=7)
        assert (r["bad"], r["good"], r["none"]) == (ref.bad, ref.good, ref.none)
        bad = np.flatnonzero(rows[c]["feedback"] == 2)[:3]
        assert r["badExamples"] == [7 + int(q) for q in bad]
    pos = cf.sparse_bad_positions(C, T)
    dims = cf.sparse_bad_dims(orc.gen_dims(0x5EED0C30, 0, C, 0, T, 300, 2), pos)
    for c, r in enumerate(oc.cand_dims(dims, idx_base=(1 << 40) + 8)):
        assert r["bad"] == len(pos[c]) and all(q >= T // 2 for q in pos[c])
        want = [(1 << 40) + 8 + q for q in pos[c][:3]]
        assert r["badExamples"] == want + [-1] * (3 - len(want))
