"""Per-candidate corpus reports without a GPU: the addon's job core (tests/c/jobs_candidate_corpus_test.c), the TypeScript
decoder's stride pinned to the ctypes mirror of apo_corpus_report, and the service wiring (candidateReport with byMode,
problem patterns and toolStats; runBeamSearch(rolloutRecords=...)) on hand-built reports."""
import ctypes
import importlib
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INC = ["-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "napi")]


def test_job_core_validates_and_allocates_the_corpus_reports(apo, tmp_path):
    apo.build_library()
    exe = str(tmp_path / "jobs_candidate_corpus_test")
    lib_dir = os.path.dirname(apo.LIB_PATH)
    subprocess.check_call(["gcc", "-std=c11", "-O1", "-Wall", "-Wextra", *INC, os.path.join(ROOT, "tests", "c", "jobs_candidate_corpus_test.c"),
                           os.path.join(ROOT, "napi", "apo_jobs.c"), "-L", lib_dir, "-lapo_b200", f"-Wl,-rpath,{lib_dir}", "-lpthread", "-lm", "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout + r.stderr


def test_abi_flag_symbol_and_ts_stride(apo):
    eng = importlib.import_module("senweaver-ide_b200.engine")
    assert eng.SCORE_CANDIDATE_CORPUS == 0x10 and "apo_candidate_corpus_reports" in eng.ABI_SYMBOLS
    assert ctypes.sizeof(eng.CorpusReport) == 784
    src = open(os.path.join(ROOT, "ts", "candidateReportCodec.ts")).read()
    assert f"const CORPUS_REPORT_BYTES = {ctypes.sizeof(eng.CorpusReport)};" in src
    assert "decodeCorpusReport(buf.slice(base, base + CORPUS_REPORT_BYTES))" in src
    codec = open(os.path.join(ROOT, "ts", "traceRecordCodec.ts")).read()          # the decoder the helper delegates to reads 784 bytes
    assert "new DataView(buf.buffer.buffer, buf.buffer.byteOffset, 784)" in codec
    napi = open(os.path.join(ROOT, "napi", "apo_napi.c")).read()
    assert '"candidateCorpus"' in napi and "APO_SCORE_CANDIDATE_CORPUS" in napi
    for f in ("apoScoringService.ts", "apoScoringMainService.ts"):
        assert "candidateCorpus" in open(os.path.join(ROOT, "ts", f)).read(), f


def corpus_report(eng, total, good, bad, modes, pats, tools=(10, 7, 3)):
    """modes: {mode index: (total, good, bad)}; pats: {pattern: (count, flag, severity, examples)}"""
    r = eng.CorpusReport()
    r.total, r.good, r.bad, r.none = total, good, bad, total - good - bad
    r.goodRate = good / (good + bad) if good + bad else 0.0
    for m, (t, g, b) in modes.items():
        r.byMode[m][0], r.byMode[m][1], r.byMode[m][2] = t, g, b
        r.byModeGoodRate[m] = g / (g + b) if g + b else 0.0
    r.withReward, r.rewardSum, r.avgReward = total, 0.1 * total, 0.1
    for i in range(9):
        r.dim[i].count, r.dim[i].sum, r.dim[i].avg = total, 0.5 * total, 0.5
    for p, (n, flag, sev, ex) in pats.items():
        q = r.pat[p]
        q.count, q.flag, q.severity = n, flag, sev
        for k in range(3):
            q.examples[k] = ex[k] if k < len(ex) else -1
    r.toolCalls, r.toolSucc, r.toolFail = tools
    r.toolSuccessRate = tools[1] / tools[0] if tools[0] else float("nan")
    return r


def strip(x):
    if isinstance(x, dict):
        return {k: strip(v) for k, v in x.items() if k != "id"}
    if isinstance(x, list):
        return [strip(v) for v in x]
    return x


def test_candidate_report_patterns_modes_and_tools(apo):
    eng = importlib.import_module("senweaver-ide_b200.engine")
    svc_mod = importlib.import_module("senweaver-ide_b200.apo_service")
    svc = svc_mod.APOService(None, None)
    before = list(svc._suggestions)
    cc = (eng.CorpusReport * 2)()
    # candidate 0: P4 (llmCalls > 2) emitted at high severity, P1 emitted at medium, P3 below its minimum; 'agent' mode at 1 / 6
    cc[0] = corpus_report(eng, 20, 6, 10, {1: (14, 5, 4), 2: (6, 1, 5)},
                          {3: (40, 1, 2, [2, 9, 11]), 0: (3, 1, 1, [1, 4, 5]), 2: (2, 0, 1, [7, 8])})
    # candidate 1: nothing emitted, every mode healthy, no tool call
    cc[1] = corpus_report(eng, 10, 9, 1, {1: (10, 9, 1)}, {}, tools=(0, 0, 0))
    res = eng.ScoreResult(np.array([0.1, 0.1]), np.array([20, 10], np.uint64), np.array([0], np.int32), None, None, None, cc)
    rep = svc.candidateReport(res, 0)
    assert [p["description"] for p in rep["patterns"]] == [svc_mod.PATTERN_TEXT[0][0], svc_mod.PATTERN_TEXT[3][0]]
    assert [(p["frequency"], p["severity"], p["examples"]) for p in rep["patterns"]] == [(3, "medium", [1, 4, 5]), (40, "high", [2, 9, 11])]
    assert rep["byMode"] == {"normal": {"total": 14, "good": 5, "bad": 4, "goodRate": 5 / 9},
                             "agent": {"total": 6, "good": 1, "bad": 5, "goodRate": 1 / 6}}
    assert rep["toolStats"] == {"totalToolCalls": 10, "totalToolSucceeded": 7, "totalToolFailed": 3, "toolSuccessRate": 0.7}
    sugg = [s["description"] for s in rep["suggestions"]]
    assert any(s.startswith("High-frequency issue: " + svc_mod.PATTERN_TEXT[3][0]) and "occurred 40 times" in s for s in sugg)   # APO:830-843
    assert not any(svc_mod.PATTERN_TEXT[0][0] in s for s in sugg)                                    # medium: no suggestion
    assert "agent mode approval rate is only 16.7%" in sugg and not any(s.startswith("normal mode") for s in sugg)   # APO:846-859
    assert "badExamples" not in rep                                                                  # no breakdown in this result
    quiet = svc.candidateReport(res, 1)
    assert quiet["patterns"] == [] and quiet["toolStats"]["toolSuccessRate"] is None
    assert not any("mode approval" in s["description"] for s in quiet["suggestions"])
    assert svc._suggestions == before                                                                # pure

    # without candidate_corpus the report is what the breakdown alone gives
    cands = (eng.CandidateReport * 1)()
    b = cands[0]
    b.total, b.good, b.bad, b.none, b.goodRate, b.withReward, b.rewardSum, b.avgReward = 10, 2, 6, 2, 0.25, 10, 3.0, 0.3
    for i in range(9):
        b.dim[i].count, b.dim[i].sum, b.dim[i].avg = 10, 5.0, 0.5
    b.badExamples[0], b.badExamples[1], b.badExamples[2] = 1, 4, -1
    plain = eng.ScoreResult(np.array([0.3]), np.array([10], np.uint64), np.array([0], np.int32), None, None, cands)
    got = svc.candidateReport(plain, 0)
    assert set(got) == {"candidate", "totalRollouts", "goodFeedbackCount", "badFeedbackCount", "noFeedbackCount", "goodRate", "avgReward",
                        "rewardByDimension", "patterns", "suggestions", "badExamples"}
    assert strip(got["suggestions"]) == strip(svc._generateLocalSuggestions(0.25, got["patterns"], {}, 0.3, b))
    assert got["patterns"] == [] and got["badExamples"] == [1, 4]


class _FakeRecordEngine:
    """Scripted rollout scoring: candidate c scores 0.1 * c; with candidate_corpus=True every candidate's report emits P4."""

    def __init__(self, eng_mod):
        self.m, self.calls = eng_mod, []

    def rollouts_upload(self, recs):
        assert recs.dtype == self.m.RECORD_DTYPE and recs.ndim == 2

    def score(self, C, K, source=0, candidates=False, candidate_corpus=False):
        self.calls.append((source, candidates, candidate_corpus))
        scores = np.array([0.1 * c for c in range(C)])
        topk = np.argsort(-scores, kind="stable")[:K].astype(np.int32)
        cands = (self.m.CandidateReport * C)() if candidates else None
        cc = None
        if candidate_corpus:
            cc = (self.m.CorpusReport * C)()
            for c in range(C):
                cc[c] = corpus_report(self.m, 10, 2, 8, {2: (10, 2, 8)}, {3: (8, 1, 2, [0, 1, 2])})
        return self.m.ScoreResult(scores, np.full(C, 10, np.uint64), topk, None, None, cands, cc)


def test_report_aware_beam_search_on_records(apo):
    eng = importlib.import_module("senweaver-ide_b200.engine")
    svc_mod = importlib.import_module("senweaver-ide_b200.apo_service")
    fake = _FakeRecordEngine(eng)
    svc = svc_mod.APOService(fake, None)
    seen = []

    def propose(parent, n, report=None):
        seen.append((parent["version"], report))
        return [parent["content"] + f"/{k}" for k in range(n)]

    records = lambda cands: np.zeros((len(cands), 3), eng.RECORD_DTYPE)
    svc.runBeamSearch("seed", propose, rolloutRecords=records, rounds=2, withReports=True)
    assert seen[0] == ("v0", None)
    later = [r for _, r in seen[1:]]
    assert later and all(r["patterns"][0]["description"] == svc_mod.PATTERN_TEXT[3][0] and r["byMode"]["agent"]["total"] == 10 for r in later)
    assert fake.calls and all(c == (1, True, True) for c in fake.calls)
    fake.calls.clear()
    svc.runBeamSearch("seed", lambda parent, n: ["x"] * n, rolloutRecords=records, rounds=1)
    assert fake.calls == [(1, False, False)]                                  # no reports asked: no flags
    with pytest.raises(ValueError):
        svc.runBeamSearch("seed", propose, rolloutDims=lambda c: None, rolloutRecords=records)
    with pytest.raises(ValueError):
        svc.runBeamSearch("seed", propose)
