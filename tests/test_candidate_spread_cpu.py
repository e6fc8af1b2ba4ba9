"""The per-candidate reward spread without a GPU: every fixture of tests/spread_fixtures.py reaches the edge it states, the
model's exact sums agree with an independent sum over fractions, M >= 0, the struct layout matches the header (ctypes and the
TypeScript decoder), and the beam service's spread rules hold on hand-built results."""
import ctypes
import importlib
import math
import os
from fractions import Fraction

import numpy as np
import pytest

import spread_fixtures as sf
from extremes_fixtures import final_rewards

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def fraction_sums(fr, ok):
    """(n, S1, S2) from Fractions: each term is round(fr * 2^52) to the nearest integer, ties to even"""
    xs = [round(Fraction(float(f)) * 2 ** 52) for f, k in zip(np.asarray(fr).tolist(), np.asarray(ok).tolist()) if k]
    return len(xs), sum(xs), sum(x * x for x in xs)


@pytest.mark.parametrize("recip", [False, True])
def test_model_sums_agree_with_fractions(orc, recip):
    for name, dims, w in sf.all_fixtures():
        fr, ok = final_rewards(dims, w, recip)
        for c, m in enumerate(sf.spread_model(fr, ok)):
            assert (m["n"], m["S1"], m["S2"]) == fraction_sums(fr[c], ok[c]), (name, c)
            assert m["M"] >= 0


def test_fixtures_reach_their_edges(orc):
    T = sf.const512().shape[1]
    for c, v in enumerate((-512.0, sf.F32_BELOW_512)):
        m = sf.model(sf.const512()[c:c + 1], sf.w_one())[0]
        assert m == sf.constant_model(T, v) and m["M"] == 0 and m["n"] >= 4096
        assert int(v * sf.FX) ** 2 * (T // 32) > 2 ** 128                 # one lane's sum inside one run passes 2^128
        assert all(math.copysign(1.0, m[f]) == 1.0 and m[f] == 0.0 for f in ("variance", "stdDev", "stdErr"))
    assert int(-512.0 * sf.FX) == -2 ** 61
    m2 = sf.model(sf.const2(), sf.w_one())
    assert all(mm["M"] == 0 and mm["variance"] == 0.0 for mm in m2)
    assert int(sf.F32_BELOW_2 * sf.FX) ** 2 > 2 ** 64 and ((1 << 22) + 3) * int(sf.F32_BELOW_2 * sf.FX) ** 2 > 2 ** 128

    d = sf.one_unit()
    fr, ok = final_rewards(d, sf.w_one_unit())
    x = sf.terms(fr[0], ok[0])
    assert sorted(set(x.tolist())) == [int(1.5 * sf.FX) - 1, int(1.5 * sf.FX)] and int((x != x.max()).sum()) == 1
    m = sf.spread_model(fr, ok)[0]
    assert m["M"] == m["n"] - 1 and m["S2"] > 2 ** 105 * (m["n"] - 1)

    got = {}
    for (name, mm, p, q), row in zip(sf.RN_CASES, sf.model(sf.rn_edges(), sf.w_one())):
        M = row["M"]
        assert M == p * q * mm * mm and (row["n"], row["S1"]) == (p + q, p * mm)
        b = M.bit_length()
        ulp = 1 << (b - 53)
        keep, rest = M >> (b - 53), M & (ulp - 1)
        got[name] = (rest > ulp // 2) - (rest < ulp // 2), keep & 1, int(float(M)) > M
    assert got == {"tie_even_down": (0, 0, False), "tie_up": (0, 1, True), "sticky_above": (1, 0, True), "below_half": (-1, 1, False)}

    c = sf.model(sf.counts(), sf.w_one())
    assert [r["n"] for r in c[:3]] == [0, 1, 2]
    assert math.isnan(c[0]["mean"]) and all(math.isnan(c[k][f]) for k in (0, 1) for f in ("variance", "stdDev", "stdErr"))
    assert not math.isnan(c[1]["mean"]) and c[2]["variance"] > 0
    T = sf.counts().shape[1]
    assert c[3]["n"] < T and c[4]["n"] == T and c[5]["n"] == T - 1
    for r in (c[4], c[5]):
        n = r["n"]
        assert r["S2"] == n * 2 ** 104 and r["variance"] == (float(n * n - r["S1"] ** 2 // 2 ** 104) / n) / (n - 1)
    n5 = c[5]["n"]                                                      # an even count: S1 = 0, variance = RN(RN(n) / (n - 1))
    assert c[5]["S1"] == 0 and c[5]["variance"] == (float(n5 * n5) / n5) / (n5 - 1) == n5 / (n5 - 1)
    assert sorted(d.shape[1] % 1024 for d in sf.tails()) == sorted(sf.TAILS)


def test_fields_rounding_sequence():
    m = sf.fields(3, 3 * 5, 3 * 25 + 1)                                 # M = 3 (3 * 25 + 1) - 225 = 3
    assert m["M"] == 3 and m["variance"] == (math.ldexp(3.0, -104) / 3.0) / 2.0
    assert m["stdErr"] == math.sqrt(m["variance"] / 3.0) and m["stdDev"] == math.sqrt(m["variance"])
    assert m["mean"] == math.ldexp(15.0, -52) / 3.0
    neg = sf.fields(2, -(2 ** 70) - 1, 2 ** 140)
    assert (neg["sumHi"] << 64) + neg["sumLo"] == -(2 ** 70) - 1 and 0 <= neg["sumLo"] < 2 ** 64


def test_struct_layout_and_the_ts_decoder(apo):
    eng = importlib.import_module("senweaver-ide_b200.engine")
    S = eng.CandidateSpread
    assert ctypes.sizeof(S) == 88 and eng.SCORE_CANDIDATE_SPREAD == 0x80
    assert "apo_candidate_spread" in eng.ABI_SYMBOLS
    offs = {"n": 0, "sumLo": 8, "sumHi": 16, "sumSq": 24, "mean": 48, "rewardSumSq": 56, "variance": 64, "stdDev": 72, "stdErr": 80}
    assert {f: getattr(S, f).offset for f in offs} == offs
    hdr = open(os.path.join(ROOT, "include", "apo_b200.h")).read()
    assert "#define APO_SCORE_CANDIDATE_SPREAD 0x80u" in hdr and "};                        /* 88 bytes */" in hdr
    s = S()
    s.sumLo, s.sumHi = 2 ** 64 - 5, -1
    s.sumSq[0], s.sumSq[1], s.sumSq[2] = 1, 2, 3
    assert s.sum == -5 and s.sum_sq == 1 + (2 << 64) + (3 << 128)
    src = open(os.path.join(ROOT, "ts", "candidateReportCodec.ts")).read()
    pins = {"CANDIDATE_SPREAD_BYTES": ctypes.sizeof(S), "OFF_SPR_N": S.n.offset, "OFF_SPR_SUM_LO": S.sumLo.offset,
            "OFF_SPR_SUM_HI": S.sumHi.offset, "OFF_SPR_SUM_SQ": S.sumSq.offset, "OFF_SPR_MEAN": S.mean.offset,
            "OFF_SPR_REWARD_SUM_SQ": S.rewardSumSq.offset, "OFF_SPR_VARIANCE": S.variance.offset, "OFF_SPR_STD_DEV": S.stdDev.offset,
            "OFF_SPR_STD_ERR": S.stdErr.offset}
    for name, value in pins.items():
        assert f"const {name} = {value};" in src, (name, value)
    assert "export function decodeCandidateSpread(buf: VSBuffer, C: number): CandidateSpread[]" in src
    for f in ("apoScoringService.ts", "apoScoringMainService.ts"):
        assert "candidateSpread" in open(os.path.join(ROOT, "ts", f)).read(), f
    napi = open(os.path.join(ROOT, "napi", "apo_napi.c")).read()
    assert '"candidateSpread"' in napi and napi.count("APO_SCORE_CANDIDATE_SPREAD") >= 3


class _FakeEngine:
    """Returns a scripted ScoreResult: candidate c scores 0.1 * c; its breakdown, and its spread when asked for it"""

    def __init__(self, eng_mod):
        self.m, self.calls = eng_mod, []

    def dims_upload(self, dims):
        self.C = dims.shape[0]

    def score(self, C, K, source=0, candidates=False, spread=False):
        self.calls.append((candidates, spread))
        scores = np.array([0.1 * c for c in range(C)])
        topk = np.argsort(-scores, kind="stable")[:K].astype(np.int32)
        cands = (self.m.CandidateReport * C)() if candidates else None
        for c in range(C if candidates else 0):
            r = cands[c]
            r.total, r.good, r.bad, r.none = 10, 2, 6, 2
            r.goodRate, r.withReward, r.rewardSum, r.avgReward = 0.25, 10, scores[c] * 10, scores[c]
        spr = None
        if spread:
            spr = (self.m.CandidateSpread * C)()
            for c in range(C):
                s = spr[c]
                s.n = 1 if c == 0 else 10
                s.mean, s.variance = scores[c], float("nan") if c == 0 else 0.04 * c
                s.stdDev = float("nan") if c == 0 else math.sqrt(s.variance)
                s.stdErr = float("nan") if c == 0 else math.sqrt(s.variance / 10)
        return self.m.ScoreResult(scores, np.full(C, 10, np.uint64), topk, None, None, cands, spread=spr)


def test_candidate_report_spread_and_beam_search(apo):
    svc_mod = importlib.import_module("senweaver-ide_b200.apo_service")
    fake = _FakeEngine(importlib.import_module("senweaver-ide_b200.engine"))
    svc = svc_mod.APOService(fake, None)
    res = svc.evaluateBeam([{"version": f"v{c}", "content": str(c)} for c in range(4)], dims=np.zeros((4, 6, 9), np.float32),
                           reports=True, spread=True)
    assert fake.calls == [(True, True)]
    rep = svc.candidateReport(res, 2)
    assert rep["rewardStdDev"] == math.sqrt(0.08) and rep["scoreStdErr"] == math.sqrt(0.08 / 10)
    rep0 = svc.candidateReport(res, 0)
    assert rep0["rewardStdDev"] is None and rep0["scoreStdErr"] is None
    plain = svc.candidateReport(fake.score(4, 2, candidates=True), 2)
    assert set(rep) - set(plain) == {"rewardStdDev", "scoreStdErr"}
    assert svc.getBeamState()["beam"][0]["version"] == "v3"                # adoption still by the means alone

    seen = []

    def propose(parent, n, report=None):
        seen.append(report)
        return [parent["content"] + f"/{k}" for k in range(n)]

    fake.calls.clear()
    svc.runBeamSearch("seed", propose, lambda cands: np.zeros((len(cands), 6, 9), np.float32), rounds=2, withReports=True,
                      withSpread=True)
    assert fake.calls and all(c == (True, True) for c in fake.calls)
    assert seen[0] is None and all("scoreStdErr" in r and "rewardStdDev" in r for r in seen[1:])
    fake.calls.clear()
    svc.runBeamSearch("seed", propose, lambda cands: np.zeros((len(cands), 6, 9), np.float32), rounds=1, withReports=True)
    assert fake.calls == [(True, False)]                                  # default: no spread requested


def test_spread_needs_reports(apo):
    svc_mod = importlib.import_module("senweaver-ide_b200.apo_service")
    svc = svc_mod.APOService(_FakeEngine(importlib.import_module("senweaver-ide_b200.engine")), None)
    with pytest.raises(ValueError):
        svc.runBeamSearch("seed", lambda p, n: [], lambda c: np.zeros((len(c), 6, 9), np.float32), rounds=1, withSpread=True)
