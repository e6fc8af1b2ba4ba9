"""The per-candidate extremes at the JS-reachable boundary: the addon's job core (validation, allocation, execution through the
C ABI) driven by tests/c/jobs_candidate_extremes_test.c, the addon and both TypeScript services carrying the option, and the
TypeScript decoder's hard-coded offsets pinned to the ctypes mirror of struct apo_candidate_extremes."""
import ctypes
import importlib
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INC = ["-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "napi")]


def _build(apo, tmp_path):
    apo.build_library()
    exe = str(tmp_path / "jobs_candidate_extremes_test")
    lib_dir = os.path.dirname(apo.LIB_PATH)
    subprocess.check_call(["gcc", "-std=c11", "-O1", "-Wall", "-Wextra", *INC, os.path.join(ROOT, "tests", "c", "jobs_candidate_extremes_test.c"),
                           os.path.join(ROOT, "napi", "apo_jobs.c"), "-L", lib_dir, "-lapo_b200", f"-Wl,-rpath,{lib_dir}", "-lpthread", "-lm", "-o", exe])
    return exe


def test_job_core_validates_and_allocates_the_extremes(apo, tmp_path):
    r = subprocess.run([_build(apo, tmp_path)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_job_core_returns_the_engine_extremes(apo, tmp_path):
    r = subprocess.run([_build(apo, tmp_path), "gpu"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout + r.stderr


def test_addon_and_services_carry_the_option():
    napi = open(os.path.join(ROOT, "napi", "apo_napi.c")).read()
    assert '"candidateExtremes"' in napi and napi.count("APO_SCORE_CANDIDATE_EXTREMES") >= 3    # scoreResident, score / records, tuples
    main = open(os.path.join(ROOT, "ts", "apoScoringMainService.ts")).read()
    assert main.count("!!candidateExtremes") == 3 and "r.candidateExtremes" in main                 # score, scoreTuples, scoreHostRecords
    svc = open(os.path.join(ROOT, "ts", "apoScoringService.ts")).read()
    assert "candidateExtremes?: VSBuffer" in svc and "candidateExtremes?: 0 | 1" in svc and svc.count(", candidateExtremes)") == 3


def test_ts_extremes_codec_offsets_match_the_c_struct(apo):
    eng = importlib.import_module("senweaver-ide_b200.engine")
    X = eng.CandidateExtremes
    src = open(os.path.join(ROOT, "ts", "candidateReportCodec.ts")).read()
    pins = {"EXTREMES_BYTES": ctypes.sizeof(X), "EXTREMES_N": eng.EXTREMES_N, "OFF_EXT_N": X.n.offset, "OFF_LOWEST": X.lowest.offset,
            "OFF_LOWEST_REWARD": X.lowestReward.offset, "OFF_HIGHEST": X.highest.offset, "OFF_HIGHEST_REWARD": X.highestReward.offset}
    for name, value in pins.items():
        assert f"const {name} = {value};" in src, (name, value)
    assert "export function decodeCandidateExtremes(buf: VSBuffer, c: number)" in src
