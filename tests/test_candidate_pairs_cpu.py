"""The paired comparison's model, fixtures, struct and service rules without a GPU: every fixture reaches the edge it names, the
model's integers equal an exact rational sum, the ctypes struct matches the C header's, and the beam service maps a round's
children to their parents and reports vsReference with its None rules."""
import ctypes
import importlib
import math
import os

import numpy as np
import pytest

import pair_fixtures as pf
import spread_fixtures as sf
from extremes_fixtures import final_rewards

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("name", [f[0] for f in pf.all_fixtures()])
def test_model_sums_agree_with_fractions(name):
    _, dims, refs, w = next(f for f in pf.all_fixtures() if f[0] == name)
    fr, ok = final_rewards(dims, w)
    for c, m in enumerate(pf.pair_model(fr, ok, refs)):
        if m["ref"] == pf.NONE:
            assert m["n"] == 0 and math.isnan(m["meanDiff"])
            continue
        assert (m["D1"], m["D2"]) == pf.fraction_sums(fr, ok, c, m["ref"]), c
        assert m["M"] >= 0 and m["wins"] + m["losses"] + m["ties"] == m["n"]
        assert m["n"] + m["candOnly"] == int(ok[c].sum()) and m["n"] + m["refOnly"] == int(ok[m["ref"]].sum())


def test_extreme_reaches_its_edges():
    n = (1 << 22) + 3
    m, mirror, self_ = pf.constant_pair(n, sf.F32_BELOW_512, -512.0, 1), pf.constant_pair(n, -512.0, sf.F32_BELOW_512, 0), \
        pf.constant_pair(n, -512.0, -512.0, 1)
    d = (1 << 62) - (1 << 37)
    assert m["D1"] == n * d and m["D1"] > 2 ** 83 and m["D2"] > 2 ** 128 and m["wins"] == n
    assert mirror["D1"] == -m["D1"] and mirror["losses"] == n and mirror["D2"] == m["D2"] and mirror["variance"] == m["variance"] == 0.0
    assert self_["ties"] == n and self_["D1"] == self_["D2"] == 0
    # the small extreme runs through the model itself: each term is the constant pair's
    small = pf.model(pf.extreme(8192 + 5), [1, 0], sf.w_one())
    assert small[0]["D1"] == (8192 + 5) * d and small[0]["D2"] > 2 ** 128 and small[1]["D1"] == -small[0]["D1"]


def test_one_unit_is_the_smallest_win_and_loss():
    m = pf.model(pf.one_unit(), pf.ONE_UNIT_REFS, sf.w_one_unit())
    assert (m[0]["wins"], m[0]["losses"], m[0]["D1"], m[0]["D2"]) == (1, 0, 1, 1)
    assert (m[1]["wins"], m[1]["losses"], m[1]["D1"], m[1]["D2"]) == (0, 1, -1, 1)
    assert (m[2]["wins"], m[2]["losses"], m[2]["D1"], m[2]["D2"]) == (1, 1, 0, 2)


def test_rn_edges_meet_the_four_roundings():
    m = pf.model(pf.rn_edges(), pf.RN_REFS, sf.w_one())
    for (name, mm, p, q), x in zip(sf.RN_CASES, m):
        assert x["M"] == p * q * mm * mm and x["n"] == p + q and x["refOnly"] == sf.RN_T - p - q, name
        assert x["M"].bit_length() > 53, name                  # RN(M) rounds
    assert m[4]["ref"] == pf.NONE


def test_counts_and_nulls():
    m = pf.model(pf.counts(), pf.COUNT_REFS, sf.w_one())
    assert [x["n"] for x in m] == [0, 1, 2, 0]
    assert math.isnan(m[0]["meanDiff"]) and math.isnan(m[1]["variance"]) and not math.isnan(m[2]["variance"])
    assert m[3]["candOnly"] == pf.counts().shape[1] and m[0]["refOnly"] == pf.counts().shape[1]
    for d in pf.nulls():
        fr, ok = final_rewards(d)
        assert not ok[0, -1] and ok[1, -1] and not ok[1, 0]
        x = pf.pair_model(fr, ok, pf.NULL_REFS)
        assert x[0]["refOnly"] >= 1 and x[0]["candOnly"] >= 1 and x[0]["n"] > 0


def test_shapes():
    refs = pf.SHAPE_REFS
    assert sum(int(r) == 0 for r in refs) == 3 and refs[4] == 5 and refs[5] == 6 and refs[7] == 7
    m = pf.model(pf.shapes(), refs)
    assert m[7]["ties"] == m[7]["n"] > 0 and m[7]["D1"] == 0
    assert m[0]["ref"] == m[6]["ref"] == pf.NONE


def test_struct_layout(apo):
    eng = importlib.import_module("senweaver-ide_b200.engine")
    P = eng.CandidatePair
    assert ctypes.sizeof(P) == 128 and eng.SCORE_CANDIDATE_PAIRS == 0x100 and eng.PAIR_NONE == 0xFFFFFFFF
    assert {"apo_candidate_refs_upload", "apo_candidate_pairs"} <= set(eng.ABI_SYMBOLS)
    offs = {"ref": 0, "pad": 4, "n": 8, "wins": 16, "losses": 24, "ties": 32, "candOnly": 40, "refOnly": 48, "sumLo": 56, "sumHi": 64,
            "sumSq": 72, "meanDiff": 96, "variance": 104, "stdDev": 112, "stdErr": 120}
    assert {f: getattr(P, f).offset for f in offs} == offs
    hdr = open(os.path.join(ROOT, "include", "apo_b200.h")).read()
    assert "#define APO_SCORE_CANDIDATE_PAIRS 0x100u" in hdr and "#define APO_PAIR_NONE 0xFFFFFFFFu" in hdr
    assert "};                        /* 128 bytes */" in hdr
    p = P()
    p.sumLo, p.sumHi = 2 ** 64 - 5, -1
    p.sumSq[0], p.sumSq[1], p.sumSq[2] = 1, 2, 3
    assert p.sum == -5 and p.sum_sq == 1 + (2 << 64) + (3 << 128)
    src = open(os.path.join(ROOT, "ts", "candidateReportCodec.ts")).read()
    pins = {"CANDIDATE_PAIR_BYTES": ctypes.sizeof(P), "PAIR_NONE": 0xFFFFFFFF, "OFF_PR_REF": P.ref.offset, "OFF_PR_N": P.n.offset,
            "OFF_PR_WINS": P.wins.offset, "OFF_PR_LOSSES": P.losses.offset, "OFF_PR_TIES": P.ties.offset,
            "OFF_PR_CAND_ONLY": P.candOnly.offset, "OFF_PR_REF_ONLY": P.refOnly.offset, "OFF_PR_SUM_LO": P.sumLo.offset,
            "OFF_PR_SUM_HI": P.sumHi.offset, "OFF_PR_SUM_SQ": P.sumSq.offset, "OFF_PR_MEAN_DIFF": P.meanDiff.offset,
            "OFF_PR_VARIANCE": P.variance.offset, "OFF_PR_STD_DEV": P.stdDev.offset, "OFF_PR_STD_ERR": P.stdErr.offset}
    for name, value in pins.items():
        want = f"0x{value:X}" if name == "PAIR_NONE" else str(value)
        assert f"const {name} = {want};" in src, (name, value)
    assert "export function decodeCandidatePairs(buf: VSBuffer, C: number): CandidatePair[]" in src
    for f in ("apoScoringService.ts", "apoScoringMainService.ts"):
        t = open(os.path.join(ROOT, "ts", f)).read()
        assert "candidatePairs" in t and "candidateRefsUpload" in t, f
    napi = open(os.path.join(ROOT, "napi", "apo_napi.c")).read()
    assert '"candidatePairs"' in napi and '"candidateRefsUpload"' in napi and napi.count("APO_SCORE_CANDIDATE_PAIRS") >= 3


class _FakeEngine:
    """Returns a scripted ScoreResult: candidate c scores 0.1 * c; its breakdown, and its pairs when asked for them"""

    def __init__(self, eng_mod):
        self.m, self.calls, self.refs = eng_mod, [], []

    def dims_upload(self, dims):
        self.C = dims.shape[0]

    def candidate_refs_upload(self, refs):
        self.refs.append([int(r) for r in refs])

    def score(self, C, K, source=0, candidates=False, pairs=False):
        self.calls.append((candidates, pairs))
        scores = np.array([0.1 * c for c in range(C)])
        topk = np.argsort(-scores, kind="stable")[:K].astype(np.int32)
        cands = (self.m.CandidateReport * C)() if candidates else None
        for c in range(C if candidates else 0):
            r = cands[c]
            r.total, r.good, r.bad, r.none = 10, 2, 6, 2
            r.goodRate, r.withReward, r.rewardSum, r.avgReward = 0.25, 10, scores[c] * 10, scores[c]
        prs = None
        if pairs:
            prs = (self.m.CandidatePair * C)()
            refs = self.refs[-1]
            for c in range(C):
                x = prs[c]
                x.ref = refs[c]
                if refs[c] == self.m.PAIR_NONE:
                    x.meanDiff = x.variance = x.stdDev = x.stdErr = float("nan")
                    continue
                x.n = c % 3                                       # 0, 1, 2: the None rules
                x.wins, x.ties = x.n, 0
                x.meanDiff = float("nan") if x.n == 0 else 0.01 * c
                x.stdErr = float("nan") if x.n < 2 else 0.002 * c
        return self.m.ScoreResult(scores, np.full(C, 10, np.uint64), topk, None, None, cands, pairs=prs)


def test_candidate_report_vs_reference():
    svc_mod = importlib.import_module("senweaver-ide_b200.apo_service")
    eng = importlib.import_module("senweaver-ide_b200.engine")
    fake = _FakeEngine(eng)
    svc = svc_mod.APOService(fake, None)
    refs = [eng.PAIR_NONE, 0, 0, 1, 1, 2]
    res = svc.evaluateBeam([{"version": f"v{c}", "content": str(c)} for c in range(6)], dims=np.zeros((6, 6, 9), np.float32),
                           reports=True, refs=refs)
    assert fake.calls == [(True, True)] and fake.refs == [refs]
    assert svc.candidateReport(res, 0)["vsReference"] is None
    r3, r4, r5 = (svc.candidateReport(res, c)["vsReference"] for c in (3, 4, 5))
    assert r3 == {"reference": 1, "pairedRollouts": 0, "wins": 0, "losses": 0, "ties": 0, "meanRewardDiff": None, "diffStdErr": None}
    assert r4["pairedRollouts"] == 1 and r4["meanRewardDiff"] == 0.04 and r4["diffStdErr"] is None
    assert r5["pairedRollouts"] == 2 and r5["meanRewardDiff"] == 0.05 and r5["diffStdErr"] == 0.01
    plain = svc.candidateReport(fake.score(6, 2, candidates=True), 2)
    assert set(svc.candidateReport(res, 2)) - set(plain) == {"vsReference"}
    assert svc.getBeamState()["beam"][0]["version"] == "v5"                # adoption still by the means alone


def test_parent_refs_and_beam_search():
    svc_mod = importlib.import_module("senweaver-ide_b200.apo_service")
    eng = importlib.import_module("senweaver-ide_b200.engine")
    N = eng.PAIR_NONE
    cands = [{"version": "v3"}, {"version": "v1", "parentVersion": "v0"}, {"version": "v7", "parentVersion": "v3"},
             {"version": "v8", "parentVersion": "v1"}, {"version": "v9", "parentVersion": "v1"}]
    # v1 was a child of v0 in an earlier round: carried over, it names none even though v0 is gone
    assert svc_mod.APOService.parentRefs(cands, 2).tolist() == [N, N, 0, 1, 1]
    assert svc_mod.APOService.parentRefs(cands[:1] + [{"version": "v4", "parentVersion": "v2"}], 1).tolist() == [N, N]

    fake = _FakeEngine(eng)
    svc = svc_mod.APOService(fake, None)
    seen = []

    def propose(parent, n, report=None):
        seen.append((parent["version"], report))
        return [parent["content"] + f"/{k}" for k in range(n)]

    svc.runBeamSearch("seed", propose, lambda cands: np.zeros((len(cands), 6, 9), np.float32), rounds=2, withReports=True,
                      withParentComparison=True)
    bf = svc._config["branchFactor"]
    assert fake.calls and all(c == (True, True) for c in fake.calls)
    assert fake.refs[0] == [N] + [0] * bf                                  # round 1: the seed, then its children
    beam1 = len(fake.refs[1]) - bf * len([s for s in seen if s[1] is not None])
    assert fake.refs[1][:beam1] == [N] * beam1                             # round 2: the carried-over beam names none
    assert all(r is None or "vsReference" in r for _, r in seen)
    fake.calls.clear()
    svc.runBeamSearch("seed", propose, lambda cands: np.zeros((len(cands), 6, 9), np.float32), rounds=1, withReports=True)
    assert fake.calls == [(True, False)]                                  # default: no comparison requested
    with pytest.raises(ValueError):
        svc.runBeamSearch("seed", lambda p, n: [], lambda c: np.zeros((len(c), 6, 9), np.float32), rounds=1, withParentComparison=True)
