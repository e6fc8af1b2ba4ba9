"""The exact corpus report of tests/exact_report.py against oracle.report, without a GPU: both oracles count the same records,
the sequential binary64 sums stay within their rounding bound of the exact ones, dyadic corpora (where nothing rounds) agree
bit for bit, every threshold fixture lands on the side of its flag threshold it states, and check_exact misses no field."""
import math
import struct

import numpy as np
import pytest

import corpus_fixtures as cf
import exact_report as xr
from oracle import candidates
from test_gpu_candidates import boundary_records

U = 2.0 ** -53


@pytest.fixture(scope="module")
def oc(orc):
    candidates.build()
    return candidates


def corpora(orc):
    """(name, records, idx_base): generated corpora, a planted and a saturating one, threshold-boundary records"""
    out = [(f"gen{T}", orc.gen_records(0x5EED0003, orc.STREAM_CORPUS, 0, 1, base, T, 300, 8).reshape(-1), base)
           for T, base in ((1, 5), (37, 0), (1000, 0), (100_003, 1 << 33))]
    out.append(("planted", cf.planted(50_000, idx_base=12)[0], 12))
    out.append(("saturating", cf.saturating(10_000, (0, 2, 4), 2), (1 << 40) + 8))
    out.append(("boundary", boundary_records(orc, 1, 24_000).reshape(-1), 0))
    out += [(name, recs, 3) for name, recs, *_ in xr.threshold_fixtures()]
    return out


def test_both_oracles_count_the_same_records(orc, oc):
    for name, recs, base in corpora(orc):
        ref = orc.report(recs, idx_base=base)
        fx = oc.cand_records(recs[None], idx_base=base)[0]
        assert (ref.total, ref.good, ref.bad, ref.none, ref.withReward) == tuple(fx[f] for f in ("total", "good", "bad", "none", "withReward")), name
        assert [ref.dim[i].count for i in range(9)] == [fx["dim"][i]["count"] for i in range(9)], name
        want = xr.exact_report(recs, base)
        rounded = (".sum", ".avg", "rewardSum", "avgReward") + xr.DIM_FLAGS + ("severity",)   # sequential sums, their flags
        assert all(f.endswith(rounded) for f, _, _ in xr.diff_exact(ref, want)), name
        for p in range(6):                                     # counts, flags and examples; severities where a record is 'bad'
            assert (ref.pat[p].count, ref.pat[p].flag, list(ref.pat[p].examples)) == \
                   (want["pat"][p]["count"], want["pat"][p]["flag"], want["pat"][p]["examples"]), (name, p)
            if ref.bad:
                assert ref.pat[p].severity == want["pat"][p]["severity"], (name, p)


def ulp(x):
    return math.ulp(x) if x else 0.0


def test_sequential_sums_within_their_rounding_bound(orc):
    """every term lies in [-1, 1]: the sequential sum of n terms is within (n - 1) u n of the exact one, and each exact term
    rint(v 2^52) 2^-52 within 2^-53 of v; each side rounds once more"""
    for name, recs, base in corpora(orc):
        ref, want = orc.report(recs, idx_base=base), xr.exact_report(recs, base)
        pairs = [(ref.rewardSum, want["rewardSum"], ref.avgReward, want["avgReward"], ref.withReward)]
        pairs += [(ref.dim[i].sum, want["dim"][i]["sum"], ref.dim[i].avg, want["dim"][i]["avg"], ref.dim[i].count) for i in range(9)]
        for k, (s, e, a, ea, n) in enumerate(pairs):
            if n == 0:
                assert s == e == 0.0 or (k == 0 and math.isnan(a) and math.isnan(ea)), (name, k)
                continue
            bound = (n - 1) * U * n + n * U + ulp(s) + ulp(e)
            assert abs(s - e) <= bound, (name, k, s, e)
            assert abs(a - ea) <= bound / n + ulp(a) + ulp(ea), (name, k, a, ea)


@pytest.mark.parametrize("T", [37, 4096, 100_003])
def test_dyadic_corpora_agree_bit_for_bit(orc, T):
    recs = xr.dyadic(T, seed=T)
    ref = orc.report(recs, idx_base=9, w=xr.DYADIC_W)
    assert ref.bad and all(ref.dim[i].count == ref.withReward == T for i in range(9))
    xr.check_exact(ref, xr.exact_report(recs, 9, w=xr.DYADIC_W), f"dyadic {T}")


def test_threshold_fixtures_land_where_they_state(orc):
    seen = set()
    for name, recs, dim, edge, side, flags in xr.threshold_fixtures():
        d = xr.exact_report(recs)["dim"][dim]
        assert {"at": d["avg"] == edge, "below": d["avg"] < edge, "above": d["avg"] > edge}[side], (name, d["avg"])
        assert tuple(d[f] for f in xr.DIM_FLAGS) == flags, name
        seen.add((edge, side))
        big = xr.exact_report(xr.padded(recs, (1 << 20) + 1))       # the digest's size: the same dimension, bit for bit
        assert big["dim"] == xr.exact_report(recs)["dim"], name
    assert {(-0.5, "at"), (-0.5, "below"), (-0.3, "below"), (0.0, "at"), (0.0, "below")} <= seen
    # where the sequential binary64 sum sits on the other side: the cases a tolerance could not tell apart
    fx = {name: (recs, dim) for name, recs, dim, *_ in xr.threshold_fixtures()}
    for name in ("d4_-0.3_x5", "d8_-0.3_x5", "d8_-0.3_x6"):
        recs, dim = fx[name]
        ref = orc.report(recs).dim[dim]
        assert ref.avg == -0.3 and ref.low_flag == 0, name
        assert xr.exact_report(recs)["dim"][dim]["avg"] == np.nextafter(-0.3, -1.0), name
    recs, dim = fx["d6_0.6_-0.6"]
    ref = orc.report(recs).dim[dim]
    assert ref.avg < 0.0 and ref.sugg_flag == 1
    assert xr.exact_report(recs)["dim"][dim]["fx"] == 0


def test_check_exact_misses_no_field(orc):
    """one unit in the last place of any binary64 field, any integer, flag, severity or example, and NaN against a number
    all fail; NaN against the same NaN passes"""
    recs = xr.dyadic(4096, seed=1)
    ref = orc.report(recs, w=xr.DYADIC_W)
    want = xr.exact_report(recs, w=xr.DYADIC_W)
    xr.check_exact(ref, want)
    flip = lambda x: struct.unpack("<d", struct.pack("<q", struct.unpack("<q", struct.pack("<d", x))[0] ^ 1))[0]
    edits = [lambda r: setattr(r, "avgReward", flip(r.avgReward)), lambda r: setattr(r, "rewardSum", flip(r.rewardSum)),
             lambda r: setattr(r, "goodRate", flip(r.goodRate)), lambda r: setattr(r, "toolSuccessRate", math.nan),
             lambda r: r.byModeGoodRate.__setitem__(3, flip(r.byModeGoodRate[3])), lambda r: r.byMode[0].__setitem__(2, r.byMode[0][2] + 1),
             lambda r: setattr(r, "toolFail", r.toolFail + 1), lambda r: setattr(r, "none", r.none + 1)]
    for i in range(9):
        for f in ("sum", "avg"):
            edits.append(lambda r, i=i, f=f: setattr(r.dim[i], f, flip(getattr(r.dim[i], f))))
        for f in ("count",) + xr.DIM_FLAGS:
            edits.append(lambda r, i=i, f=f: setattr(r.dim[i], f, getattr(r.dim[i], f) ^ 1))
    for p in range(6):
        for f in ("count", "flag", "severity"):
            edits.append(lambda r, p=p, f=f: setattr(r.pat[p], f, getattr(r.pat[p], f) ^ 1))
        for k in range(3):
            edits.append(lambda r, p=p, k=k: r.pat[p].examples.__setitem__(k, r.pat[p].examples[k] + 1))
    for e in edits:
        r = orc.report(recs, w=xr.DYADIC_W)
        e(r)
        assert len(xr.diff_exact(r, want)) == 1
        with pytest.raises(AssertionError):
            xr.check_exact(r, want)
    none = np.repeat(xr.record(feedback=2, flags=0, toolCalls=0, toolSucc=0), 5)   # no reward, no tool call: both NaN
    xr.check_exact(orc.report(none), xr.exact_report(none))
