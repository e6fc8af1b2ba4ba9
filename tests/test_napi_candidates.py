"""The per-candidate breakdown at the JS-reachable boundary: the addon's job core (validation, allocation, execution through
the C ABI) driven by tests/c/jobs_candidates_test.c, and the TypeScript decoder's hard-coded offsets pinned to the ctypes
mirror of apo_candidate_report."""
import ctypes
import importlib
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INC = ["-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "napi")]


def _build(apo, tmp_path):
    apo.build_library()
    exe = str(tmp_path / "jobs_candidates_test")
    lib_dir = os.path.dirname(apo.LIB_PATH)
    subprocess.check_call(["gcc", "-std=c11", "-O1", "-Wall", "-Wextra", *INC, os.path.join(ROOT, "tests", "c", "jobs_candidates_test.c"),
                           os.path.join(ROOT, "napi", "apo_jobs.c"), "-L", lib_dir, "-lapo_b200", f"-Wl,-rpath,{lib_dir}", "-lpthread", "-lm", "-o", exe])
    return exe


def test_job_core_validates_and_allocates_the_breakdown(apo, tmp_path):
    r = subprocess.run([_build(apo, tmp_path)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_job_core_returns_the_engine_breakdown(apo, tmp_path):
    r = subprocess.run([_build(apo, tmp_path), "gpu"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout + r.stderr


def test_addon_and_services_carry_the_candidates_option():
    src = open(os.path.join(ROOT, "napi", "apo_napi.c")).read()
    assert '"candidates"' in src and "APO_SCORE_CANDIDATES" in src
    for f in ("apoScoringService.ts", "apoScoringMainService.ts"):
        ts = open(os.path.join(ROOT, "ts", f)).read()
        assert "candidates" in ts, f


def test_ts_candidate_codec_offsets_match_the_c_struct(apo):
    """ts/candidateReportCodec.ts hard-codes the byte layout of apo_candidate_report; pin it to the ctypes mirror."""
    eng = importlib.import_module("senweaver-ide_b200.engine")
    R, D = eng.CandidateReport, eng.DimStat
    off = {f: getattr(R, f).offset for f, _ in R._fields_}
    src = open(os.path.join(ROOT, "ts", "candidateReportCodec.ts")).read()
    pins = {"CANDIDATE_REPORT_BYTES": ctypes.sizeof(R), "OFF_TOTAL": off["total"], "OFF_GOOD": off["good"], "OFF_BAD": off["bad"],
            "OFF_NONE": off["none"], "OFF_GOOD_RATE": off["goodRate"], "OFF_WITH_REWARD": off["withReward"], "OFF_REWARD_SUM": off["rewardSum"],
            "OFF_AVG_REWARD": off["avgReward"], "OFF_DIM": off["dim"], "DIMSTAT_BYTES": ctypes.sizeof(D), "OFF_BAD_EXAMPLES": off["badExamples"],
            "DIM_COUNT": D.count.offset, "DIM_AVG": D.avg.offset, "DIM_LOW_FLAG": D.low_flag.offset, "DIM_LOW_SEVERITY": D.low_severity.offset,
            "DIM_SUGG_FLAG": D.sugg_flag.offset, "DIM_SUGG_PRIORITY": D.sugg_priority.offset}
    for name, value in pins.items():
        assert f"const {name} = {value};" in src, (name, value)
