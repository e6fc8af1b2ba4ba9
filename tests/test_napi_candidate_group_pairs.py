"""The paired comparisons per record group at the JS-reachable boundary: the addon's job core (validation, allocation,
execution through the C ABI) driven by tests/c/jobs_candidate_group_pairs_test.c."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INC = ["-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "napi")]


def _build(apo, tmp_path):
    apo.build_library()
    exe = str(tmp_path / "jobs_candidate_group_pairs_test")
    lib_dir = os.path.dirname(apo.LIB_PATH)
    subprocess.check_call(["gcc", "-std=c11", "-O1", "-Wall", "-Wextra", "-Werror", *INC,
                           os.path.join(ROOT, "tests", "c", "jobs_candidate_group_pairs_test.c"), os.path.join(ROOT, "napi", "apo_jobs.c"),
                           "-L", lib_dir, "-lapo_b200", f"-Wl,-rpath,{lib_dir}", "-lpthread", "-lm", "-o", exe])
    return exe


def test_job_core_validates_and_allocates_the_group_pairs(apo, tmp_path):
    r = subprocess.run([_build(apo, tmp_path)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_job_core_returns_the_engine_group_pairs(apo, tmp_path):
    r = subprocess.run([_build(apo, tmp_path), "gpu"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout + r.stderr
