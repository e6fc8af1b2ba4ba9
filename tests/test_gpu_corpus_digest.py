"""The corpus digest on the H100 (-m gpu): for a corpus of at least 2^20 records, the second scoring call with a corpus report
after the load counts the distinct reward keys of its VALID records and keeps the words of the corpus block that no weight
reaches (csrc/apo_kernels.h CorpusDigestParams); that call and the later ones that would scan the resident corpus stand-alone
derive their corpus words from them instead (k_corpus_digest), and K1h runs the same pass and the tail inside its own launch.
Every report on the digest route must be byte-equal to the scan route of the same engine (TUNE_NO_CORPUS_DIGEST set after
the load) and field-equal to the CPU oracle: the benchmark's 5 M corpus, the planted and saturating corpora of
tests/corpus_fixtures.py at both idx_base values, weights set after the load, recip, the K1h / K1t2 / resident Form T routes,
sessions finished repeatedly, a host-streaming call, a reload; K1h in one launch at forced grids of 1, 2, 3 and 7 CTAs over the
5 M corpus's digest; a corpus reported once builds nothing; corpora the gate refuses build nothing and scan.  The 36 M-record flush cases of
tests/test_gpu_corpus_flush.py run again with no digest, so that k_detect6_tiles keeps their coverage."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import corpus_fixtures as cf
import corpus_digest_model as dm
import test_gpu_corpus_flush as flush
import test_gpu_count_route as cr
from test_gpu_candidate_corpus import check_oracle

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

SEED = 0x5EED0003
BENCH_T = 5_000_000
BASES = (0, (1 << 40) + 8)
W_CUSTOM = np.array([0.3, 0.1, 0.05, 0.05, 0.1, 0.1, 0.1, 0.1, 0.1])
W_ZERO = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])   # masks without d5 weigh 0: null
SAT = ((0, 2, 4), 2)


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(autouse=True)
def restore(engine, apo, orc):
    engine.set_tuning(0)
    w0 = orc.weights()
    yield
    engine.set_tuning(0)
    engine.set_weights(w0)


def both_routes(engine, apo, call, flags=0):
    """call() on the digest route, then with TUNE_NO_CORPUS_DIGEST set after the load (the scan): the same report bytes"""
    engine.set_tuning(flags)
    a = call()
    engine.set_tuning(flags | apo.TUNE_NO_CORPUS_DIGEST)
    b = call()
    engine.set_tuning(flags)
    assert bytes(a.report) == bytes(b.report)
    assert np.array_equal(a.scores, b.scores) and np.array_equal(a.topk, b.topk)
    return a


def small_dims(orc):
    return orc.gen_dims(0x5EED0C31, 0, 3, 0, 4096, 300, 2)


def warm(engine, call):
    """the load is followed by one reported call: no digest yet; the second builds it"""
    call()
    assert engine.debug_corpus_digest() is None
    call()


def check_digest(engine, orc, recs, idx_base):
    """the entries are the model's, the fixed words the scan's (the oracle's report)"""
    got = engine.debug_corpus_digest()
    assert got is not None
    ent, fixed = got
    assert sorted(map(tuple, ent.tolist())) == dm.entries(recs)
    assert [int(x) for x in fixed] == dm.fixed_words(orc.report(recs, idx_base=idx_base, nthreads=16), idx_base)


def test_bench_corpus(engine, apo, orc):
    """the benchmark's corpus (seed 0x5EED0003, 5 M records) under default, custom and zero weights and recip"""
    engine.corpus_generate(SEED, 0, BENCH_T, 300)
    engine.set_tuning(apo.TUNE_TWIN_T)
    engine.dims_upload(small_dims(orc))
    warm(engine, lambda: engine.score(3, 1, corpus=True))
    got = engine.debug_corpus_digest()
    assert got is not None and 0 < len(got[0]) <= min(1 << 20, BENCH_T // 4)
    for w in (None, W_CUSTOM, W_ZERO):
        if w is not None:
            engine.set_weights(w)
        ref = orc.report_generated(SEED, 0, BENCH_T, w=w)
        for recip in (False, True):
            r = both_routes(engine, apo, lambda: engine.score(3, 1, corpus=True, recip=recip), apo.TUNE_TWIN_T)
            check_oracle(apo, r.report, ref)
    assert engine.debug_corpus_digest() is not None        # set_weights keeps the digest


@pytest.mark.parametrize("idx_base", BASES)
@pytest.mark.parametrize("kind", ["planted", "saturating"])
def test_fixture_corpora(engine, apo, orc, kind, idx_base):
    T = (1 << 21) + 3
    if kind == "saturating":
        recs, want = cf.saturating(T, *SAT), None
    else:
        recs, _, want = cf.planted(T, idx_base=idx_base)
    engine.corpus_upload(recs, idx_base)
    engine.dims_upload(small_dims(orc))
    engine.set_tuning(apo.TUNE_NO_FUSE)
    warm(engine, lambda: engine.score(3, 1, corpus=True))
    check_digest(engine, orc, recs, idx_base)
    r = both_routes(engine, apo, lambda: engine.score(3, 1, corpus=True), apo.TUNE_NO_FUSE)
    ref = orc.report(recs, idx_base=idx_base, nthreads=16)
    if kind == "saturating":
        flush.check_oracle_ints(r.report, ref)
        cf.check_closed_form(r.report, cf.closed_form(T, *SAT, idx_base=idx_base))
    else:
        check_oracle(apo, r.report, ref)
        cf.check_designed(r.report, want)


def test_routes_sessions_and_reload(engine, apo, orc):
    """K1h (one launch), K1t2, resident Form T, sessions finished twice, host streaming; then a reload replaces the digest"""
    recs = orc.gen_records(0x5EED0D16, orc.STREAM_CORPUS, 0, 1, 0, 1 << 20, 300).reshape(-1)
    engine.corpus_upload(recs, 17)
    ref = orc.report(recs, idx_base=17, nthreads=16)
    dims = cr.build()
    engine.set_tuning(apo.TUNE_TWIN_T)
    engine.dims_upload(dims)
    assert engine.debug_twin_h() is not None                                        # whole rows read through K1h
    warm(engine, lambda: engine.score(cr.C, 2, corpus=True))
    check_digest(engine, orc, recs, 17)
    for corpus in (True, False):                                                   # the digest pass + tail, or the tail alone
        r = engine.score(cr.C, 2, corpus=corpus)
        assert r.timing.launches == 1
    for flags in (apo.TUNE_TWIN_T, apo.TUNE_TWIN_T | apo.TUNE_NO_TWIN_H):        # K1h, K1t2
        check_oracle(apo, both_routes(engine, apo, lambda: engine.score(cr.C, 2, corpus=True), flags).report, ref)

    def session():
        engine.score_begin(cr.C)
        engine.score_accumulate(0)
        first = engine.score_finish(cr.C, 2, corpus=True)
        engine.score_accumulate(0)
        second = engine.score_finish(cr.C, 2, corpus=True)
        assert bytes(first.report) == bytes(second.report)
        return second
    check_oracle(apo, both_routes(engine, apo, session, apo.TUNE_TWIN_T).report, ref)
    engine.dims_tuples()
    check_oracle(apo, both_routes(engine, apo, lambda: engine.score(cr.C, 2, source=apo.SRC_TUPLES, corpus=True), apo.TUNE_TWIN_T).report, ref)
    host = np.ascontiguousarray(small_dims(orc))
    check_oracle(apo, both_routes(engine, apo, lambda: engine.score_host(host, 2, corpus=True), apo.TUNE_TWIN_T).report, ref)
    recs2 = cf.saturating((1 << 20) + 5, *SAT)                                        # reload: the new corpus's digest
    engine.corpus_upload(recs2, 0)
    warm(engine, lambda: engine.score(cr.C, 2, corpus=True))
    check_digest(engine, orc, recs2, 0)
    r = both_routes(engine, apo, lambda: engine.score(cr.C, 2, corpus=True), apo.TUNE_TWIN_T)
    cf.check_closed_form(r.report, cf.closed_form(len(recs2), *SAT, idx_base=0))


def test_gate_builds_nothing(engine, apo, orc):
    """more than 2^20 distinct d2 keys, or fewer than 2^20 records: no digest, the scan, the oracle's report; a corpus reported
    once, or with TUNE_NO_CORPUS_DIGEST set, builds none"""
    many = dm.distinct_d2(1 << 22, seed=0x5EED0D17)
    few = orc.gen_records(0x5EED0D18, orc.STREAM_CORPUS, 0, 1, 0, (1 << 20) - 1, 300).reshape(-1)
    engine.dims_upload(small_dims(orc))
    for recs in (many, few):
        engine.corpus_upload(recs, 5)
        for _ in range(3):
            r = engine.score(3, 1, corpus=True)
            assert engine.debug_corpus_digest() is None
        check_oracle(apo, r.report, orc.report(recs, idx_base=5, nthreads=16))
    engine.corpus_generate(SEED, 0, 1 << 21, 300)
    engine.score(3, 1, corpus=True)                                                    # reported once: nothing built
    assert engine.debug_corpus_digest() is None
    engine.set_tuning(apo.TUNE_NO_CORPUS_DIGEST)
    engine.score(3, 1, corpus=True)
    engine.score(3, 1, corpus=True)
    assert engine.debug_corpus_digest() is None


GRID_SCRIPT = r"""
import importlib, json, sys
sys.path[:0] = [sys.argv[1], sys.argv[2]]
import test_gpu_count_route as cr
apo = importlib.import_module("senweaver-ide_b200")
e = apo.Engine(0)
e.set_tuning(apo.TUNE_TWIN_T)
e.dims_upload(cr.build())
e.corpus_generate(int(sys.argv[3]), 0, int(sys.argv[4]), 300)
out = {}
for _ in range(3):
    r = e.score(cr.C, 2, corpus=True)
out["entries"] = len(e.debug_corpus_digest()[0])
out["launches"] = int(r.timing.launches)
out["digest"] = bytes(r.report).hex()
out["scores"] = r.scores.tolist()
e.set_tuning(apo.TUNE_TWIN_T | apo.TUNE_NO_CORPUS_DIGEST)
out["scan"] = bytes(e.score(cr.C, 2, corpus=True).report).hex()
e.close()
print(json.dumps(out))
"""


def test_k1h_one_launch_forced_grids(engine, apo, orc):
    """K1h with the digest pass and the tail in its launch, at 1, 2, 3 and 7 CTAs (APO_K1_GRID, read once per process) over
    the 5 M corpus's ~80 k entries: one launch, the scan's report bytes, the oracle's report, the same scores at every grid"""
    ref = orc.report_generated(SEED, 0, BENCH_T)
    scores = None
    for g in (1, 2, 3, 7):
        p = subprocess.run([sys.executable, "-c", GRID_SCRIPT, ROOT, HERE, str(SEED), str(BENCH_T)], env=dict(os.environ, APO_K1_GRID=str(g)),
                           capture_output=True, text=True, timeout=600)
        assert p.returncode == 0, p.stderr[-3000:]
        out = json.loads(p.stdout.strip().splitlines()[-1])
        assert out["entries"] > 7 * 1024 and out["launches"] == 1, (g, out["entries"], out["launches"])
        assert out["digest"] == out["scan"], g
        check_oracle(apo, apo.engine.CorpusReport.from_buffer_copy(bytes.fromhex(out["digest"])), ref)
        assert scores is None or out["scores"] == scores
        scores = out["scores"]


@pytest.mark.parametrize("kind,idx_base", [("saturating", flush.BIG_BASE), ("planted", 0)])
def test_36M_flush_cases_without_digest(engine, orc, apo, sm_count, kind, idx_base):
    """the 36 M-record cases of test_gpu_corpus_flush with the digest off at the load: every host scans the records"""
    engine.set_tuning(apo.TUNE_NO_CORPUS_DIGEST)
    flush.test_36M_corpus_through_every_scan_host(_NoDigest(engine, apo), orc, apo, sm_count, kind, idx_base)


class _NoDigest:
    """the engine with TUNE_NO_CORPUS_DIGEST kept under every tuning the flush test sets"""
    def __init__(self, e, apo):
        self._e, self._flag = e, apo.TUNE_NO_CORPUS_DIGEST

    def set_tuning(self, flags):
        self._e.set_tuning(flags | self._flag)

    def corpus_upload(self, recs, idx_base=0):
        self._e.corpus_upload(recs, idx_base)
        assert self._e.debug_corpus_digest() is None

    def __getattr__(self, name):
        return getattr(self._e, name)
