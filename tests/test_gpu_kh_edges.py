"""K1h (k_reward9th) at the edges of its launch (-m gpu), on the fixtures of tests/kh_fixtures.py.

The search tensors put the CTA cuts of forced grids of 2, 3, 7 and 13 CTAs and of the default grid on the probe offsets of
every round of the ballot search and one pair either side, inside the last row and inside one row under every CTA; the
stride tensors give rows and row remainders of 7936 +- 1 and 15 873 pairs (992 streaming threads beside the digest warp)
and 8192 +- 1 (1024 threads); the digest tensors, at 7 CTAs, uneven and zero digest shares and launches whose CTAs take
both digest passes, at 128 * share - 1, 128 * share and 128 * share + 1 pairs.  One process per grid (APO_K1_GRID is read
once per process).  The K3 cases run C = 1 ... 4096 rows with tie groups and -inf rows through K1h's finalising tail,
which ranks by counting up to C = 1024 and selects by radix from 1025 on.

For every tensor the counts the load built must be count_model's, and on each path -- the call without a corpus report
(the tail rides on K1h: 992 streaming threads), the call with a corpus report from the digest (one launch), a session
score_begin / score_accumulate(0) / score_finish (1024 threads, the stand-alone tail) and TUNE_NO_FUSE -- the integers must
be the oracle's, the scores bit-equal to sharding.scores_from_partials and the top-K sharding.topk_indices, with the same
bytes as the engine under TUNE_NO_TWIN_H (K1t2 / K1t).  Corpus reports must be byte-equal to the scan's
(TUNE_NO_CORPUS_DIGEST) and to the stand-alone k_corpus_digest's, and field-equal to the oracle's.  No tolerance anywhere.

The module took 40 s on one H100 80GB HBM3 at 700 W."""
import importlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import count_model as cm
import k1_fixtures as kf
import kh_fixtures as kh
import test_gpu_count_route as cr
from test_gpu_candidate_corpus import check_oracle

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sharding = importlib.import_module("senweaver-ide_b200.sharding")
PATHS = ("tail", "digest", "session", "nofuse")


def call(e, apo, path, C, K, extra=0):
    """one call of `path` under TUNE_TWIN_T | extra: (result, integers)"""
    tw = apo.TUNE_TWIN_T | extra
    if path == "session":
        e.set_tuning(tw)
        e.score_begin(C)
        e.score_accumulate(0)
        r = e.score_finish(C, K)
    else:
        e.set_tuning(tw | (apo.TUNE_NO_FUSE if path == "nofuse" else 0))
        r = e.score(C, K, corpus=path in ("digest", "nofuse"))
    return r, e.debug_partials(C)


def check_counts(e, dims, off):
    got = e.debug_twin_h()
    assert got is not None
    C, T = dims.shape[:2]
    assert np.array_equal(got[0].astype(np.int64), off)
    want_off, want_pairs = cm.pairs(cr.indices(e, C, T), T)
    assert np.array_equal(got[0], want_off) and np.array_equal(got[1], want_pairs)


def check_paths(e, apo, name, C, K, want, ref, nkeys):
    """every path: the oracle's integers, scores and top-K from them, the same bytes under TUNE_NO_TWIN_H; reports equal to
    the scan's, the stand-alone digest pass's and the oracle's"""
    scores = sharding.scores_from_partials(*want)
    topk = sharding.topk_indices(scores, K)
    try:
        for path in PATHS:
            for _ in range(3):                                   # a corpus reported once builds no digest yet
                r, p = call(e, apo, path, C, K)
                if path != "digest" or r.timing.launches == 1:
                    break
            where = (name, path, C, K)
            assert p == want, where
            assert r.scores.tobytes() == scores.tobytes() and r.counts.tolist() == want[1], where
            assert np.array_equal(r.topk, topk), where
            if path in ("tail", "digest"):
                assert r.timing.launches == 1, where
            r2, p2 = call(e, apo, path, C, K, apo.TUNE_NO_TWIN_H)
            assert p2 == p and r2.scores.tobytes() == r.scores.tobytes() and np.array_equal(r2.topk, r.topk), where
            if r.report is not None:
                dig = e.debug_corpus_digest()
                assert dig is not None and len(dig[0]) == nkeys, where
                scan, _ = call(e, apo, path, C, K, apo.TUNE_NO_CORPUS_DIGEST)
                assert bytes(r.report) == bytes(r2.report) == bytes(scan.report), where
                check_oracle(apo, r.report, ref)
    finally:
        e.set_tuning(apo.TUNE_TWIN_T)


def run_grid():
    """every search and stride tensor (and at DIG_GRID the digest tensors) at the grid of this process's APO_K1_GRID"""
    import oracle as orc
    apo = importlib.import_module("senweaver-ide_b200")
    grid = int(os.environ.get("APO_K1_GRID", "0")) or None
    e = apo.Engine(0)
    done = []
    try:
        e.set_tuning(apo.TUNE_TWIN_T)
        recs = kh.digest_corpus(kh.ROW_KEYS)
        e.corpus_upload(recs, kh.IDX_BASE)
        ref = orc.report(recs, idx_base=kh.IDX_BASE, nthreads=16)
        for fx in kh.search_fixtures() + kh.stride_fixtures():
            dims = kh.fixture_dims(fx)
            e.set_tuning(apo.TUNE_TWIN_T)
            e.dims_upload(dims)
            check_counts(e, dims, fx.off)
            check_paths(e, apo, fx.name, dims.shape[0], fx.K, orc.score_dims_fx(dims), ref, kh.ROW_KEYS)
            done.append(fx.name)
        if grid == kh.DIG_GRID:
            for fx in kh.digest_fixtures():
                dims = kh.fixture_dims(fx)
                e.set_tuning(apo.TUNE_TWIN_T)
                e.dims_upload(dims)
                check_counts(e, dims, fx.off)
                want = orc.score_dims_fx(dims)
                for n in kh.DIG_KEYS:
                    recs = kh.digest_corpus(n)
                    e.set_tuning(apo.TUNE_TWIN_T)
                    e.corpus_upload(recs, kh.IDX_BASE)
                    check_paths(e, apo, f"{fx.name}/{n}", dims.shape[0], fx.K, want,
                                orc.report(recs, idx_base=kh.IDX_BASE, nthreads=16), n)
                    done.append(f"{fx.name}/{n}")
    finally:
        e.close()
    print(json.dumps(done))


@pytest.mark.parametrize("grid", kh.GRIDS)
def test_kh_edges_at_grid(grid):
    env = dict(os.environ)
    env.pop("APO_K1_GRID", None)
    if grid:
        env["APO_K1_GRID"] = str(grid)
    p = subprocess.run([sys.executable, "-c", "import sys; sys.path[:0] = [sys.argv[1], sys.argv[2]]; "
                        "import test_gpu_kh_edges as t; t.run_grid()", ROOT, HERE],
                       env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-4000:]
    done = json.loads(p.stdout.strip().splitlines()[-1])
    names = [fx.name for fx in kh.search_fixtures() + kh.stride_fixtures()]
    if grid == kh.DIG_GRID:
        names += [f"{fx.name}/{n}" for fx in kh.digest_fixtures() for n in kh.DIG_KEYS]
    assert done == names


@pytest.fixture(scope="module")
def k3_corpus(engine, apo, orc):
    engine.set_tuning(apo.TUNE_TWIN_T)
    recs = kh.digest_corpus(kh.ROW_KEYS)
    engine.corpus_upload(recs, kh.IDX_BASE)
    yield orc.report(recs, idx_base=kh.IDX_BASE, nthreads=16)
    engine.set_tuning(0)


@pytest.mark.parametrize("C,mode", kh.k3_cases())
def test_k3_through_k1h(engine, apo, orc, k3_corpus, C, mode):
    dims = kh.k3_dims(C, mode)
    engine.set_tuning(apo.TUNE_TWIN_T)
    engine.dims_upload(dims)
    check_counts(engine, dims, kh.k3_offsets(C, mode))
    want = orc.score_dims_fx(dims)
    for K in kf.k_values(kf.scores_of(*want)):
        check_paths(engine, apo, f"k3/{mode}", C, K, want, k3_corpus, kh.ROW_KEYS)
