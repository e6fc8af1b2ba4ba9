"""The per-candidate group scores on the CPU: the two models of tests/group_fixtures.py agree on every fixture, the groups of
a candidate add up to its scoring integers, every fixture reaches the edge it is built for, the ctypes mirror of
apo_group_score has the header's layout and the TypeScript decoder's offsets, and the beam service builds byGroup and
refuses malformed groups."""
import ctypes
import importlib
import math
import os

import numpy as np
import pytest

import group_fixtures as gf
import k1_fixtures as kf
from extremes_fixtures import final_rewards, record_final_rewards

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def same(a, b) -> bool:
    """score tables equal, binary64 fields compared as bit patterns (NaN included)"""
    def key(s):
        return tuple(np.float64(v).tobytes() if isinstance(v, float) else v for v in s.values())
    return [[key(s) for s in row] for row in a] == [[key(s) for s in row] for row in b]


def fixtures():
    return gf.all_fixtures() + [("wide",) + gf.wide() + (gf.w_d0(),)]


@pytest.mark.parametrize("recip", [False, True])
@pytest.mark.parametrize("name", [f[0] for f in fixtures()])
def test_models_agree_and_add_up_to_the_scoring_integers(orc, name, recip):
    _, dims, labels, G, w = next(f for f in fixtures() if f[0] == name)
    fr, ok = final_rewards(dims, w, recip)
    tally = gf.dims_tally(dims)
    a, b = gf.group_model(fr, ok, tally, labels, G), gf.group_model_split(fr, ok, tally, labels, G)
    assert same(a, b)
    sums, counts = kf.fx_model(dims, w=w, recip=recip)
    for c in range(dims.shape[0]):
        assert sum(s["sum"] for s in a[c]) == sums[c] and sum(s["withReward"] for s in a[c]) == counts[c]
        assert sum(s["total"] for s in a[c]) == dims.shape[1]


def test_records_add_up_to_the_scoring_integers(orc):
    recs = orc.gen_records(0x5EED6100, orc.STREAM_ROLLOUT, 0, 2, 0, 700, 300, 4)
    recs["flags"][:, ::5] &= ~np.uint8(8)
    labels = (np.arange(700) // 7 % 5).astype(np.uint8)
    m = gf.rec_model(recs, labels, 5)
    fr, ok = record_final_rewards(recs)
    assert same(m, gf.group_model_split(fr, ok, gf.record_tally(recs), labels, 5))
    sums, counts = orc.score_records_fx(recs)
    for c in range(2):
        assert sum(s["sum"] for s in m[c]) == sums[c] and sum(s["withReward"] for s in m[c]) == counts[c]
        # tallies from the feedback field, VALID or not
        assert sum(s["bad"] for s in m[c]) == int((recs["feedback"][c] == 2).sum())


def test_g1_is_the_breakdown(orc):
    dims, labels, G = gf.zero()
    m = gf.model(dims, labels, G)
    sums, counts = kf.fx_model(dims)
    for c in range(dims.shape[0]):
        s = m[c][0]
        assert s["sum"] == sums[c] and s["withReward"] == counts[c] and s["total"] == dims.shape[1]
        assert s["avgReward"] == (float(sums[c]) / 2 ** 52) / counts[c]


def test_fixtures_reach_their_edges(orc):
    _, labels, G = gf.mod(64)
    assert G == 64 and np.all(np.diff(labels.astype(int)) != 0)               # a new label on every record
    _, labels, _ = gf.edges()
    t = np.nonzero(np.diff(labels.astype(int)))[0] + 1                        # first record of every new run
    assert set(t % 32) == {0, 31} and {1024, 2048, 3072, 4096, 5120} <= set(t.tolist())
    for r in gf.TAILS:
        dims, labels, G = gf.last(r)
        assert dims.shape[1] % 1024 == r and np.nonzero(labels == 1)[0].tolist() == [dims.shape[1] - 1]
        m = gf.model(dims, labels, G)
        assert all(row[2]["total"] == 0 and math.isnan(row[2]["avgReward"]) and row[2]["goodRate"] == 0.0 for row in m)
        assert all(row[1]["total"] == 1 for row in m)
    dims, labels, G = gf.wide()
    m = gf.model(dims, labels, G, w=gf.w_d0())
    assert all(abs(s["sum"]) > 2 ** 64 for row in m for s in row)
    assert m[0][0]["sum"] == -m[0][1]["sum"] and m[1][0]["sum"] < 0 and m[1][1]["sum"] < 0
    dims, labels, G = gf.null()
    m = gf.model(dims, labels, G, w=gf.W_NULL)
    for row in m:
        assert row[1]["withReward"] == 0 and math.isnan(row[1]["avgReward"]) and row[1]["good"] > 0 and row[1]["bad"] > 0
        assert row[0]["withReward"] > 0 and row[2]["withReward"] > 0


def test_group_score_layout_and_the_ts_decoder(apo):
    eng = importlib.import_module("senweaver-ide_b200.engine")
    S = eng.GroupScore
    assert ctypes.sizeof(S) == 56 and eng.GROUPS_MAX == 64 and eng.SCORE_CANDIDATE_GROUPS == 0x40
    assert {"apo_record_groups_upload", "apo_candidate_groups"} <= set(eng.ABI_SYMBOLS)
    src = open(os.path.join(ROOT, "ts", "candidateReportCodec.ts")).read()
    pins = {"GROUP_SCORE_BYTES": ctypes.sizeof(S), "OFF_GRP_TOTAL": S.total.offset, "OFF_GRP_GOOD": S.good.offset,
            "OFF_GRP_BAD": S.bad.offset, "OFF_GRP_GOOD_RATE": S.goodRate.offset, "OFF_GRP_WITH_REWARD": S.withReward.offset,
            "OFF_GRP_REWARD_SUM": S.rewardSum.offset, "OFF_GRP_AVG_REWARD": S.avgReward.offset}
    for name, value in pins.items():
        assert f"const {name} = {value};" in src, (name, value)
    assert "export function decodeCandidateGroups(buf: VSBuffer, C: number, G: number): GroupScore[][]" in src
    for f in ("apoScoringService.ts", "apoScoringMainService.ts"):
        ts = open(os.path.join(ROOT, "ts", f)).read()
        assert "candidateGroups" in ts and "recordGroupsUpload(" in ts, f
    napi = open(os.path.join(ROOT, "napi", "apo_napi.c")).read()
    assert '{"recordGroupsUpload", NULL,' in napi and '"candidateGroups"' in napi and napi.count("APO_SCORE_CANDIDATE_GROUPS") >= 3


class _FakeEngine:
    """Returns a scripted ScoreResult: candidate c scores 0.1 * c; its breakdown, and its group scores when asked for them"""

    def __init__(self, eng_mod):
        self.m, self.calls, self.G = eng_mod, [], 0

    def dims_upload(self, dims):
        self.C = dims.shape[0]

    def record_groups_upload(self, labels, G):
        self.labels, self.G = np.asarray(labels), G

    def score(self, C, K, source=0, candidates=False, groups=False):
        self.calls.append((candidates, groups))
        scores = np.array([0.1 * c for c in range(C)])
        topk = np.argsort(-scores, kind="stable")[:K].astype(np.int32)
        cands = (self.m.CandidateReport * C)() if candidates else None
        for c in range(C if candidates else 0):
            r = cands[c]
            r.total, r.good, r.bad, r.none = 10, 2, 6, 2
            r.goodRate, r.withReward, r.rewardSum, r.avgReward = 0.25, 10, scores[c] * 10, scores[c]
            r.badExamples[0], r.badExamples[1], r.badExamples[2] = 1, -1, -1
        grp = None
        if groups:
            grp = ((self.m.GroupScore * self.G) * C)()
            for c in range(C):
                for g in range(self.G):
                    s = grp[c][g]
                    s.total, s.good, s.bad, s.goodRate = 5 + g, 1, 2, 1 / 3
                    s.withReward = 0 if g == self.G - 1 else 4
                    s.rewardSum = 0.5 * c
                    s.avgReward = float("nan") if s.withReward == 0 else 0.125 * c
        return self.m.ScoreResult(scores, np.full(C, 10, np.uint64), topk, None, None, cands, None, None, grp)


def test_candidate_report_by_group_and_beam_search(apo):
    svc_mod = importlib.import_module("senweaver-ide_b200.apo_service")
    fake = _FakeEngine(importlib.import_module("senweaver-ide_b200.engine"))
    svc = svc_mod.APOService(fake, None)
    labels = np.array([0, 1, 2, 0, 1, 2], np.uint8)
    names = ["agent", "chat", "held-out"]

    res = svc.evaluateBeam([{"version": f"v{c}", "content": str(c)} for c in range(4)], dims=np.zeros((4, 6, 9), np.float32),
                           reports=True, groups=(labels, names))
    assert np.array_equal(fake.labels, labels) and fake.G == 3
    rep = svc.candidateReport(res, 2)
    assert rep["byGroup"] == {
        "agent": {"totalRollouts": 5, "goodFeedbackCount": 1, "badFeedbackCount": 2, "goodRate": 1 / 3, "avgReward": 0.25},
        "chat": {"totalRollouts": 6, "goodFeedbackCount": 1, "badFeedbackCount": 2, "goodRate": 1 / 3, "avgReward": 0.25},
        "held-out": {"totalRollouts": 7, "goodFeedbackCount": 1, "badFeedbackCount": 2, "goodRate": 1 / 3, "avgReward": None}}
    assert list(svc.candidateReport(res, 2, groupNames=["a", "b", "c"])["byGroup"]) == ["a", "b", "c"]
    plain = svc.candidateReport(fake.score(4, 2, candidates=True), 2)
    assert "byGroup" not in plain and set(rep) - set(plain) == {"byGroup"}

    seen = []

    def propose(parent, n, report=None):
        seen.append(report)
        return [parent["content"] + f"/{k}" for k in range(n)]

    def rollouts(cands):
        return np.zeros((len(cands), 6, 9), np.float32)

    fake.calls.clear()
    svc.runBeamSearch("seed", propose, rollouts, rounds=2, withReports=True, rolloutGroups=(labels, names))
    assert fake.calls and all(c == (True, True) for c in fake.calls)
    assert seen[0] is None and all(list(r["byGroup"]) == names for r in seen[1:])
    fake.calls.clear()
    svc.runBeamSearch("seed", propose, rollouts, rounds=1, withReports=True)
    assert fake.calls == [(True, False)]                                  # default: no group scores requested


@pytest.mark.parametrize("names", [[], ["a", "a"], [f"g{i}" for i in range(65)]])
def test_malformed_groups_are_refused(apo, names):
    svc_mod = importlib.import_module("senweaver-ide_b200.apo_service")
    fake = _FakeEngine(importlib.import_module("senweaver-ide_b200.engine"))
    svc = svc_mod.APOService(fake, None)
    labels = np.zeros(6, np.uint8)
    with pytest.raises(ValueError):
        svc.runBeamSearch("seed", lambda p, n, r=None: [], lambda c: np.zeros((len(c), 6, 9), np.float32), rounds=1,
                          withReports=True, rolloutGroups=(labels, names))
    assert svc.evaluateBeam([{"version": "v0", "content": ""}], dims=np.zeros((1, 6, 9), np.float32), reports=True,
                            groups=(labels, names)) is None and fake.calls == []


def test_groups_need_reports(apo):
    svc_mod = importlib.import_module("senweaver-ide_b200.apo_service")
    svc = svc_mod.APOService(_FakeEngine(importlib.import_module("senweaver-ide_b200.engine")), None)
    with pytest.raises(ValueError):
        svc.runBeamSearch("seed", lambda p, n: [], lambda c: np.zeros((len(c), 6, 9), np.float32), rounds=1,
                          rolloutGroups=(np.zeros(6, np.uint8), ["a"]))
