"""The dimsTuples job at the JS-reachable boundary: the addon's job core (validation of cap, FIFO order, execution through
apo_dims_tuples) driven by tests/c/jobs_tuples_test.c, and the addon and TypeScript services carrying the call."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INC = ["-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "napi")]


def _build(apo, tmp_path):
    apo.build_library()
    exe = str(tmp_path / "jobs_tuples_test")
    lib_dir = os.path.dirname(apo.LIB_PATH)
    subprocess.check_call(["gcc", "-std=c11", "-O1", "-Wall", "-Wextra", "-Werror", *INC, os.path.join(ROOT, "tests", "c", "jobs_tuples_test.c"),
                           os.path.join(ROOT, "napi", "apo_jobs.c"), "-L", lib_dir, "-lapo_b200", f"-Wl,-rpath,{lib_dir}", "-lpthread", "-lm", "-o", exe])
    return exe


def test_job_core_validates_and_orders_dims_tuples(apo, tmp_path):
    r = subprocess.run([_build(apo, tmp_path)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_job_core_builds_form_t_through_the_engine(apo, tmp_path):
    r = subprocess.run([_build(apo, tmp_path), "gpu"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout + r.stderr


def test_addon_and_services_carry_dims_tuples():
    src = open(os.path.join(ROOT, "napi", "apo_napi.c")).read()
    assert '{"dimsTuples", NULL,' in src and "APO_JOB_DIMS_TUPLES" in src
    for f in ("apoScoringService.ts", "apoScoringMainService.ts"):
        ts = open(os.path.join(ROOT, "ts", f)).read()
        assert "dimsTuples(cap?: number): Promise<number>" in ts, f
    svc = open(os.path.join(ROOT, "ts", "apoScoringService.ts")).read()
    assert "source?: 0 | 1 | 2;" in svc
