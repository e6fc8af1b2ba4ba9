"""Per-candidate breakdown without a GPU: the oracle (oracle/candidates.py) against the corpus report of the same rows
and against a plain numpy restatement, the ctypes layout of apo_candidate_report, and the service wiring
(candidateReport, runBeamSearch(withReports=True)) on a fake engine result."""
import ctypes
import importlib
import math

import numpy as np
import pytest


@pytest.fixture(scope="module")
def oc(orc):
    from oracle import candidates
    candidates.build()
    return candidates


def test_oracle_breakdown_of_record_rows_is_their_corpus_report(orc, oc):
    """A Form R candidate row is a list of traces: every shared field equals oracle.report(row) (the reference-pinned corpus
    report); integers exactly, the binary64 sums (exact there, sequential in the reference) within the pin's 1e-12."""
    recs = orc.gen_records(0x5EED0C11, orc.STREAM_ROLLOUT, 0, 4, 0, 6000, 300, 4)
    rng = np.random.default_rng(5)
    recs["flags"][rng.random(recs.shape) < 0.05] &= ~np.uint8(8)              # never-scored traces: tallied, not rewarded
    recs[3]["flags"] &= ~np.uint8(8)                                          # a row without a single reward
    for c, b in enumerate(oc.cand_records(recs)):
        ref = orc.report(recs[c])
        assert (b["total"], b["good"], b["bad"], b["none"], b["withReward"]) == (ref.total, ref.good, ref.bad, ref.none, ref.withReward)
        assert b["goodRate"] == ref.goodRate
        if ref.withReward:
            assert b["avgReward"] == pytest.approx(ref.avgReward, rel=1e-12, abs=1e-12)
            assert b["rewardSum"] == pytest.approx(ref.rewardSum, rel=1e-12, abs=1e-9)
        else:
            assert math.isnan(b["avgReward"]) and math.isnan(ref.avgReward)
        for i in range(9):
            d, r = b["dim"][i], ref.dim[i]
            assert d["count"] == r.count
            assert d["sum"] == pytest.approx(r.sum, rel=1e-12, abs=1e-9)
            assert d["avg"] == pytest.approx(r.avg, rel=1e-12, abs=1e-12)
            assert (d["low_flag"], d["sugg_flag"]) == (r.low_flag, r.sugg_flag)
        bad = np.flatnonzero(recs[c]["feedback"] == 2)[:3].tolist()
        assert b["badExamples"] == bad + [-1] * (3 - len(bad))


def numpy_breakdown(dims, w, idx_base=0):
    """Plain restatement: TCS:777-784 per row in push order, exact integer sums of rint(x * 2^52)."""
    Cn, T, _ = dims.shape
    out = []
    for c in range(Cn):
        v = dims[c].astype(np.float64)
        present = ~np.isnan(v)
        ws = np.zeros(T); tw = np.zeros(T)
        for i in range(9):
            ws = ws + np.where(present[:, i], v[:, i], 0.0) * w[i]
            tw = tw + np.where(present[:, i], w[i], 0.0)
        valid = tw > 0
        fr = np.where(valid, ws / np.where(valid, tw, 1.0), 0.0)
        d0 = v[:, 0]
        good, bad = int(np.sum(d0 == 1.0)), int(np.sum(d0 == -1.0))
        fx = sum(int(x) for x in np.rint(fr[valid] * 2.0 ** 52))
        dims_fx = []
        for i in range(9):
            m = valid & present[:, i]
            dims_fx.append((sum(int(x) for x in np.rint(v[m, i] * 2.0 ** 52)), int(m.sum())))
        ex = (np.flatnonzero(d0 == -1.0)[:3] + idx_base).tolist()
        out.append({"total": T, "good": good, "bad": bad, "withReward": int(valid.sum()), "rewardFx": fx, "dims": dims_fx,
                    "badExamples": ex + [-1] * (3 - len(ex))})
    return out


@pytest.mark.parametrize("zero_weights", [False, True])
def test_oracle_breakdown_of_dims_against_numpy(orc, oc, zero_weights):
    rng = np.random.default_rng(11 + zero_weights)
    Cn, T = 5, 3000
    dims = rng.choice(np.array([-1.0, -0.5, -0.2, 0.0, 0.3, 0.5, 0.8, 1.0], np.float32), size=(Cn, T, 9))
    dims[..., 2] = rng.random((Cn, T)).astype(np.float32) * 2 - 1
    dims[rng.random(dims.shape) < 0.2] = np.nan                                # absent dimensions
    dims[rng.random((Cn, T)) < 0.05] = np.nan                                  # null rows
    dims[2] = np.nan                                                           # an all-null candidate
    w = orc.weights().copy()
    if zero_weights:
        w[[0, 3, 5]] = 0.0                                                     # rows present only there: total weight 0 -> null
    ours = oc.cand_dims(dims, idx_base=40, w=w)
    ref = numpy_breakdown(dims, w, idx_base=40)
    for b, r in zip(ours, ref):
        assert (b["total"], b["good"], b["bad"], b["withReward"], b["rewardFx"]) == (r["total"], r["good"], r["bad"], r["withReward"], r["rewardFx"])
        assert [(d["fx"], d["count"]) for d in b["dim"]] == r["dims"]
        assert b["badExamples"] == r["badExamples"]
        for d in b["dim"]:
            assert d["sum"] == float(d["fx"]) * 2.0 ** -52 and d["avg"] == (d["sum"] / d["count"] if d["count"] else 0.0)
    assert ours[2]["withReward"] == 0 and math.isnan(ours[2]["avgReward"]) and ours[2]["total"] == T
    # the generator path (threads over record slices) gives the same as the materialised tensor
    gen = orc.gen_dims(0x5EED0C12, 3, 2, 100, 5000, 300, 4)
    assert oc.cand_dims(gen, idx_base=100) == oc.cand_generated(0x5EED0C12, [3, 4], 100, 5000, 300, nthreads=7)
    recs = orc.gen_records(0x5EED0C12, orc.STREAM_ROLLOUT, 3, 2, 100, 5000, 300, 4)
    assert oc.cand_records(recs, idx_base=100) == oc.cand_generated(0x5EED0C12, [3, 4], 100, 5000, 300, nthreads=5, records=True)


def test_candidate_report_struct_layout(apo):
    eng = importlib.import_module("senweaver-ide_b200.engine")
    R = eng.CandidateReport
    assert ctypes.sizeof(R) == 376
    off = {f: getattr(R, f).offset for f, _ in R._fields_}
    assert (off["total"], off["good"], off["bad"], off["none"], off["goodRate"], off["withReward"], off["rewardSum"], off["avgReward"],
            off["dim"], off["badExamples"]) == (0, 8, 16, 24, 32, 40, 48, 56, 64, 352)
    assert eng.SCORE_CANDIDATES == 0x8 and "apo_candidate_reports" in eng.ABI_SYMBOLS


class _FakeEngine:
    """Returns a scripted ScoreResult: candidate c scores 0.1 * c, its breakdown says d4 (tool_call_efficiency) is low."""

    def __init__(self, eng_mod):
        self.m, self.calls = eng_mod, []

    def dims_upload(self, dims):
        self.C = dims.shape[0]

    def score(self, C, K, source=0, candidates=False):
        self.calls.append(candidates)
        scores = np.array([0.1 * c for c in range(C)])
        topk = np.argsort(-scores, kind="stable")[:K].astype(np.int32)
        cands = None
        if candidates:
            cands = (self.m.CandidateReport * C)()
            for c in range(C):
                r = cands[c]
                r.total, r.good, r.bad, r.none = 10, 2, 6, 2
                r.goodRate, r.withReward, r.rewardSum, r.avgReward = 0.25, 10, scores[c] * 10, scores[c]
                for i in range(9):
                    r.dim[i].count, r.dim[i].sum, r.dim[i].avg = 10, 5.0, 0.5
                r.dim[4].sum, r.dim[4].avg, r.dim[4].low_flag, r.dim[4].low_severity = -8.0, -0.8, 1, 2
                r.dim[4].sugg_flag, r.dim[4].sugg_priority = 1, 2
                r.badExamples[0], r.badExamples[1], r.badExamples[2] = 1, 4, -1
        return self.m.ScoreResult(scores, np.full(C, 10, np.uint64), topk, None, None, cands)


def test_candidate_report_and_report_aware_beam_search(apo):
    svc_mod = importlib.import_module("senweaver-ide_b200.apo_service")
    fake = _FakeEngine(importlib.import_module("senweaver-ide_b200.engine"))
    svc = svc_mod.APOService(fake, None)
    suggestions_before = list(svc._suggestions)

    res = fake.score(5, 2, candidates=True)
    rep = svc.candidateReport(res, 3)
    assert (rep["goodFeedbackCount"], rep["badFeedbackCount"], rep["noFeedbackCount"], rep["goodRate"]) == (2, 6, 2, 0.25)
    assert rep["avgReward"] == pytest.approx(0.3) and rep["badExamples"] == [1, 4]
    assert rep["rewardByDimension"]["tool_call_efficiency"] == {"sum": -8.0, "count": 10, "avg": -0.8}
    assert [p["description"] for p in rep["patterns"]] == ["tool_call_efficiency dimension reward signal consistently low (avg: -0.800)"]
    assert any("tool_call_efficiency dimension performing poorly" in s["description"] for s in rep["suggestions"])
    assert svc._suggestions == suggestions_before                             # pure: nothing recorded

    seen = []

    def propose(parent, n, report=None):
        seen.append((parent["version"], None if report is None else report["candidate"]))
        return [parent["content"] + f"/{k}" for k in range(n)]

    svc.runBeamSearch("seed", propose, lambda cands: np.zeros((len(cands), 2, 9), np.float32), rounds=2, withReports=True)
    assert seen[0] == ("v0", None)                                            # the unscored seed has no report
    assert all(r is not None for _, r in seen[1:]) and len(seen) > 1
    assert fake.calls and all(fake.calls)

    fake.calls.clear()
    legacy = []
    svc.runBeamSearch("seed", lambda parent, n: legacy.append(parent["version"]) or ["x"] * n,
                      lambda cands: np.zeros((len(cands), 2, 9), np.float32), rounds=1)
    assert legacy == ["v0"] and fake.calls == [False]                         # defaults: no breakdown requested
