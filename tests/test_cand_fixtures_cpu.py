"""The per-candidate breakdown fixtures (tests/cand_fixtures.py) on the CPU: each reaches the edge it is built for, checked
with exact integers and fractions, and the CPU oracle (oracle/candidates.py) equals the exact pure-Python model of the
breakdown on every one of them, the refusal of values without an exact fixed-point term included.  This pins the oracle
at these edges before the GPU is compared with it (tests/test_gpu_cand_edges.py)."""
import math
import struct
from fractions import Fraction

import numpy as np
import pytest

import cand_fixtures as cf

FX = cf.FX


@pytest.fixture(scope="module")
def oc(orc):
    from oracle import candidates
    candidates.build()
    return candidates


def bits(x: float) -> bytes:
    return struct.pack("<d", x)


def canon(reps: list[dict]) -> list[dict]:
    """floats as bit patterns (NaN, -0.0 and every last bit compared)"""
    def f(x):
        return bits(x) if isinstance(x, float) else x
    return [{k: ([{kk: f(vv) for kk, vv in d.items()} for d in v] if k == "dim" else f(v)) for k, v in r.items()} for r in reps]


def oracle_or_refusal(oc, dims, w, idx_base=0):
    """(breakdowns, refused) from the oracle"""
    try:
        return oc.cand_dims(dims, w=w, idx_base=idx_base), False
    except oc.CandDomainError as e:
        return e.reports, True


def fixtures():
    yield "large_sums", cf.large_sums(), cf.W_BIG
    yield "ties", cf.ties(), cf.W_BIG
    yield "report_rules", cf.report_rules(), cf.W_BIG
    yield "tallies", cf.tallies(), cf.W_BIG
    for r in cf.SHAPE_TAILS:
        yield f"shapes_{r}", cf.shapes(r), None
    yield "many_short", cf.many_short(), None
    for v, where in cf.domain_cases():
        d, w = cf.domain(v, where)
        yield f"domain_{v:g}_{where}", d, w


@pytest.fixture(scope="module")
def large():
    d = cf.large_sums()
    return d, cf.exact_breakdown(d, cf.W_BIG)[0]


def test_large_sums_pass_2_64_and_2_83_and_cancel_across_warps(large):
    d, ref = large
    assert all(r["withReward"] >= 1 << 20 for r in ref)
    for c, s in ((0, 1), (1, -1)):
        dim = ref[c]["dim"]
        assert s * dim[3]["fx"] > 1 << 83 and dim[3]["count"] == cf.LARGE_T
        assert dim[3]["fx"] == s * cf.LARGE_T * ((1 << 63) - (1 << 39))        # the largest exact term, every evaluation
        assert -s * dim[4]["fx"] > 1 << 64
        assert s * dim[8]["fx"] > 1 << 32 and dim[8]["fx"] == s * cf.LARGE_T << 12
    for c, s in ((2, 1), (3, -1)):
        dim = ref[c]["dim"]
        assert dim[3]["fx"] == 0 and bits(dim[3]["sum"]) == bits(0.0) and dim[3]["sugg_flag"] == 0 and dim[3]["count"] > 1 << 20
        assert dim[4]["fx"] == s and dim[8]["fx"] == s << 64
        h = cf.LARGE_T // 2
        col = d[c, :, 3]
        assert (col[:h] > 0).all() and (col[h:2 * h] < 0).all()               # the halves lie ~500 tiles apart: other warps


def test_tie_sums_are_ties_in_both_branches_of_limbs_to_double():
    ref, refused = cf.exact_breakdown(cf.ties(), cf.W_BIG)
    assert not refused
    for k, (name, S) in enumerate(cf.TIE_SUMS.items()):
        for c, s in ((2 * k, 1), (2 * k + 1, -1)):
            fx = ref[c]["dim"][3]["fx"]
            assert fx == s * S, name
            e = 7 if name.startswith("lo") else 11
            assert (S < 1 << 64) == name.startswith("lo")
            exact = Fraction(fx, FX)
            if name.endswith("tie"):
                assert S == ((1 << 53) + 1) << e                               # exactly halfway between two binary64s
                assert ref[c]["dim"][3]["sum"] == s * 2.0 ** (53 + e - 52)     # ties to even: down
            else:
                assert S == (((1 << 53) + 1) << e) + 1                         # the sticky unit breaks the tie: up
                assert ref[c]["dim"][3]["sum"] == s * (2.0 ** (53 + e - 52) + 2.0 ** (e - 51))
            assert abs(Fraction(ref[c]["dim"][3]["sum"]) - exact) <= Fraction(1, 2) * 2 ** (e - 51)


def test_to_fx_ties_round_half_to_even():
    halves = [Fraction(v) * FX for v in cf.TIE_VALUES[:6]]
    assert all(h.denominator == 2 for h in halves)                             # k + 1/2
    assert [round(h) for h in halves] == [0, 2, 2, 0, -2, -2]
    sub = np.float32(cf.TIE_VALUES[6])
    assert 0 < sub < np.finfo(np.float32).tiny and round(Fraction(float(sub)) * FX) == 0
    ref, _ = cf.exact_breakdown(cf.ties(), cf.W_BIG)
    n = cf.ties().shape[1]
    per = [0, 2, 2, 0, -2, -2, 0]
    assert all(r["dim"][4]["fx"] == sum(per[t % 7] for t in range(n)) for r in ref)


def test_report_rows_reach_every_threshold_from_both_sides():
    R = cf.report_rows()
    ref, _ = cf.exact_breakdown(cf.report_rules(), cf.W_BIG)
    seen = set()
    for (vals, want), r in zip(R, ref):
        dm = r["dim"][5]
        assert dm["count"] == len(vals) and dm["avg"] == want
        seen.add((dm["count"], dm["low_flag"], dm["low_severity"], dm["sugg_flag"], dm["sugg_priority"]))
    rn03 = [(v, a) for v, a in R if a == -0.3]
    assert rn03 and all(Fraction(sum(Fraction(float(np.float32(x))) for x in v), len(v)) == Fraction(-3, 10) for v, _ in rn03)
    for t in (-0.3, -0.5):
        assert {float(np.nextafter(t, -1)), t, float(np.nextafter(t, 1))} <= {a for _, a in R}
    assert {a for _, a in R if abs(a) < 1e-15} >= {0.0} and min(a for _, a in R if abs(a) < 1e-15) < 0 < max(a for _, a in R if abs(a) < 1e-15)
    assert {n for n, *_ in seen} == {2, 3, 4, 5}
    assert {(lf, ls) for n, lf, ls, *_ in seen if n == 5} >= {(0, 1), (1, 1), (1, 2)}   # low_flag / low_severity
    assert {(sf, sp) for n, _, _, sf, sp in seen if n >= 3} >= {(0, 1), (1, 1), (1, 2)}  # sugg_flag / sugg_priority
    assert any(n == 2 and sf == 0 for n, _, _, sf, _ in seen)                 # avg < 0 under the count threshold


def test_tallies_and_good_rate_edges():
    d = cf.tallies()
    ref, _ = cf.exact_breakdown(d, cf.W_BIG)
    assert ref[0]["good"] == ref[0]["bad"] > 0 and ref[0]["goodRate"] == 0.5
    assert ref[1]["good"] == 0 < ref[1]["bad"] and ref[1]["goodRate"] == 0.0
    assert ref[2]["bad"] == 0 < ref[2]["good"] and ref[2]["goodRate"] == 1.0
    assert ref[3]["good"] == ref[3]["bad"] == 0 and ref[3]["none"] == d.shape[1] and ref[3]["goodRate"] == 0.0
    assert ref[4]["withReward"] == 0 and ref[4]["bad"] == d.shape[1] and math.isnan(ref[4]["avgReward"])
    assert ref[1]["withReward"] < d.shape[1] and ref[1]["dim"][3]["count"] == 0    # null evaluations: in no sum
    tw = sum(cf.W_BIG[[1, 2, 5, 6, 7]])
    assert tw == 1 - 2.0 ** -53 and float.hex(tw) == "0x1.fffffffffffffp-1"   # all-ones significand


def test_domain_fixtures_refuse_exactly_the_counted_values_past_2048():
    for v, where in cf.domain_cases():
        d, w = cf.domain(v, where)
        _, refused = cf.exact_breakdown(d, w)
        assert refused == cf.domain_refused(v, where), (v, where)
        assert refused == (where == "pair" or (where != "null" and v != cf.BIG))


def test_shapes_hold_their_row_ends():
    assert {cf.shapes(r).shape[1] % 1024 for r in cf.SHAPE_TAILS} == set(cf.SHAPE_TAILS)
    assert cf.many_short().shape == (600, 33, 9)


def test_every_fixture_fits_every_loader():
    """<= 15 values per coded dimension and <= 4095 tool_success_rate values: the same tensor goes through Form W / P / T"""
    for name, d, _ in fixtures():
        for i in range(9):
            col = d[..., i]
            n = len(np.unique(col[~np.isnan(col)]))
            assert n <= (4095 if i == 2 else 15), (name, i, n)


def test_oracle_equals_exact_model_on_every_fixture(oc):
    for name, d, w in fixtures():
        want, want_refused = cf.exact_breakdown(d, w)
        got, refused = oracle_or_refusal(oc, d, w)
        assert refused == want_refused, name
        assert canon(got) == canon(want), name
