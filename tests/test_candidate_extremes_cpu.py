"""The per-candidate extremes on the CPU: the fixtures (tests/extremes_fixtures.py) reach the edges they are built for, the
two models of the lists agree on every one of them, the per-evaluation rewards sum to the scoring call's exact integers,
the ctypes mirror of struct apo_candidate_extremes has the header's layout, and the beam service shapes the lists into
candidate reports as documented."""
import ctypes
import importlib
import math

import numpy as np
import pytest

import extremes_fixtures as xf
import k1_fixtures as kf


def same(a: dict, b: dict) -> bool:
    """list equality with rewards compared as bit patterns (NaN past n included)"""
    def bits(v):
        return [np.float64(x).tobytes() for x in v]
    return (a["n"] == b["n"] and a["lowest"] == b["lowest"] and a["highest"] == b["highest"]
            and bits(a["lowestReward"]) == bits(b["lowestReward"]) and bits(a["highestReward"]) == bits(b["highestReward"]))


@pytest.mark.parametrize("recip", [False, True])
@pytest.mark.parametrize("name", [f[0] for f in xf.all_fixtures()])
def test_sorted_and_inserted_lists_agree(orc, name, recip):
    _, dims, w = next(f for f in xf.all_fixtures() if f[0] == name)
    fr, ok = xf.final_rewards(dims, w, recip)
    for c in range(dims.shape[0]):
        pos = 1000 + np.arange(dims.shape[1])
        a, b = xf.extremes_sorted(fr[c], ok[c], pos), xf.extremes_inserted(fr[c], ok[c], pos)
        assert same(a, b), (name, c)
        assert a["n"] == min(32, int(ok[c].sum()))
        assert all(x >= 1000 for x in a["lowest"][:a["n"]])


@pytest.mark.parametrize("recip", [False, True])
@pytest.mark.parametrize("name", [f[0] for f in xf.all_fixtures()])
def test_rewards_are_the_scored_ones(orc, name, recip):
    """sum over the row of rint(fr * 2^52) and the count of non-null evaluations are the scoring arithmetic's (fx_model)"""
    _, dims, w = next(f for f in xf.all_fixtures() if f[0] == name)
    fr, ok = xf.final_rewards(dims, w, recip)
    sums, counts = kf.fx_model(dims, w=w, recip=recip)
    for c in range(dims.shape[0]):
        fx = np.rint(fr[c][ok[c]] * float(1 << 52)).astype(np.int64)
        assert sum(int(x) for x in fx) == sums[c] and int(ok[c].sum()) == counts[c]


def test_record_rewards_are_the_scored_ones(orc):
    recs = orc.gen_records(0x5EED3000, orc.STREAM_ROLLOUT, 0, 2, 0, 300, 300, 4)
    fr, ok = xf.record_final_rewards(recs)
    sums, counts = orc.score_records_fx(recs)
    for c in range(2):
        fx = np.rint(fr[c][ok[c]] * float(1 << 52)).astype(np.int64)
        assert sum(int(x) for x in fx) == sums[c] and int(ok[c].sum()) == counts[c]


def test_fixtures_reach_their_edges(orc):
    m = xf.model(xf.ties())
    assert all(r["n"] == 32 and r["lowest"] == list(range(32)) and r["highest"] == list(range(32)) for r in m)
    assert [r["n"] for r in xf.model(xf.counts())] == [0, 1, 31, 32, 32]
    m = xf.model(xf.null_rows(), w=xf.W_ZERO)
    assert m[0]["n"] == 0 and m[0]["lowest"] == [-1] * 32 and all(math.isnan(x) for x in m[0]["highestReward"])
    assert m[1]["n"] == 32 and m[2]["n"] == 0
    T = xf.falling().shape[1]
    m = xf.model(xf.falling())[0]
    assert m["lowest"] == list(range(T - 1, T - 33, -1)) and m["highest"] == list(range(32))
    T = xf.last().shape[1]
    m = xf.model(xf.last())[0]
    assert m["lowest"][0] == T - 1 and m["highest"][0] == T - 2 and m["lowest"][1:] == list(range(31))
    m = xf.model(xf.ulps())
    for r in m:
        assert len(set(r["lowestReward"][:24])) == 3 and r["lowestReward"][24:] == [0.0] * 8
        assert len(set(r["highestReward"][:24])) == 3 and r["highestReward"][24:] == [0.0] * 8
    assert sorted(d.shape[1] % 1024 for d in xf.tails()) == sorted(list(xf.TAILS) * 2)


def test_zero_is_reported_positive(orc):
    d = xf.rows(40, d1=np.float32(0.0))
    d[::2, 1] = -0.0
    m = xf.model(d[None])[0]
    assert all(np.float64(x).tobytes() == np.float64(0.0).tobytes() for x in m["lowestReward"])


def test_extremes_struct_layout(apo):
    eng = importlib.import_module("senweaver-ide_b200.engine")
    X = eng.CandidateExtremes
    assert ctypes.sizeof(X) == 1032 and eng.EXTREMES_N == 32
    assert (X.n.offset, X.lowest.offset, X.lowestReward.offset, X.highest.offset, X.highestReward.offset) == (0, 8, 264, 520, 776)
    assert eng.SCORE_CANDIDATE_EXTREMES == 0x20 and "apo_candidate_extremes" in eng.ABI_SYMBOLS


class _FakeEngine:
    """Returns a scripted ScoreResult: candidate c scores 0.1 * c; its breakdown, and its lists when asked for them"""

    def __init__(self, eng_mod):
        self.m, self.calls = eng_mod, []

    def dims_upload(self, dims):
        self.C = dims.shape[0]

    def score(self, C, K, source=0, candidates=False, extremes=False):
        self.calls.append((candidates, extremes))
        scores = np.array([0.1 * c for c in range(C)])
        topk = np.argsort(-scores, kind="stable")[:K].astype(np.int32)
        cands = (self.m.CandidateReport * C)() if candidates else None
        for c in range(C if candidates else 0):
            r = cands[c]
            r.total, r.good, r.bad, r.none = 10, 2, 6, 2
            r.goodRate, r.withReward, r.rewardSum, r.avgReward = 0.25, 10, scores[c] * 10, scores[c]
            r.badExamples[0], r.badExamples[1], r.badExamples[2] = 1, -1, -1
        ext = None
        if extremes:
            ext = (self.m.CandidateExtremes * C)()
            for c in range(C):
                x = ext[c]
                x.n = 3
                for i in range(32):
                    x.lowest[i] = x.highest[i] = -1
                    x.lowestReward[i] = x.highestReward[i] = float("nan")
                for i in range(3):
                    x.lowest[i], x.lowestReward[i] = 10 * c + i, -0.5 + 0.25 * i
                    x.highest[i], x.highestReward[i] = 10 * c + 9 - i, 0.75 - 0.125 * i
        return self.m.ScoreResult(scores, np.full(C, 10, np.uint64), topk, None, None, cands, None, ext)


def test_candidate_report_lists_and_beam_search(apo):
    svc_mod = importlib.import_module("senweaver-ide_b200.apo_service")
    fake = _FakeEngine(importlib.import_module("senweaver-ide_b200.engine"))
    svc = svc_mod.APOService(fake, None)

    plain = svc.candidateReport(fake.score(4, 2, candidates=True), 2)
    assert "lowestRollouts" not in plain and "highestRollouts" not in plain
    rep = svc.candidateReport(fake.score(4, 2, candidates=True, extremes=True), 2)
    assert rep["lowestRollouts"] == [{"index": 20, "finalReward": -0.5}, {"index": 21, "finalReward": -0.25},
                                     {"index": 22, "finalReward": 0.0}]
    assert rep["highestRollouts"] == [{"index": 29, "finalReward": 0.75}, {"index": 28, "finalReward": 0.625},
                                      {"index": 27, "finalReward": 0.5}]
    assert set(rep) - set(plain) == {"lowestRollouts", "highestRollouts"}
    for k in plain:                                                       # suggestions / patterns carry fresh uuids
        if k not in ("suggestions", "patterns"):
            assert rep[k] == plain[k], k
    assert [x["description"] for x in rep["suggestions"]] == [x["description"] for x in plain["suggestions"]]

    seen = []

    def propose(parent, n, report=None):
        seen.append(report)
        return [parent["content"] + f"/{k}" for k in range(n)]

    fake.calls.clear()
    svc.runBeamSearch("seed", propose, lambda cands: np.zeros((len(cands), 2, 9), np.float32), rounds=2, withReports=True,
                      withExtremes=True)
    assert fake.calls and all(c == (True, True) for c in fake.calls)
    assert seen[0] is None and all("lowestRollouts" in r and len(r["highestRollouts"]) == 3 for r in seen[1:])

    fake.calls.clear()
    svc.runBeamSearch("seed", propose, lambda cands: np.zeros((len(cands), 2, 9), np.float32), rounds=1, withReports=True)
    assert fake.calls == [(True, False)]                                  # default: no lists requested
    with pytest.raises(ValueError):
        svc.runBeamSearch("seed", propose, lambda cands: np.zeros((len(cands), 2, 9), np.float32), rounds=1, withExtremes=True)
