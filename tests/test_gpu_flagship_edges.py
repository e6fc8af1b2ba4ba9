"""The flagship step's one launch at its edges (-m gpu), on the fixtures of tests/flagship_fixtures.py.

K1h (k_reward9th) over the Form T copy's per-row dictionary counts: a dictionary at the copy's cap of 2^20 entries counted in
three batches of 64 rows (the last ragged) and one past the cap (no copy); two full batches; the chunk and thread-slice
edges of k_th_rows; both sides of the nnz gate; rows of 2^25 evaluations whose count * value products pass 2^64.  The
counts the load built must be count_model's from the copy's index planes, and every call's integers the oracle's (the numpy
model for recip) and those of the same engine under TUNE_NO_TWIN_H (K1t2 / K1t) and TUNE_NO_TWIN_T (K1q), with weights set
after the load; forced grids of 1, 2, 3 and 7 CTAs give the same bytes.

The corpus digest at its gates: exactly the cap of distinct VALID keys (kept) and one more (dropped) at caps 2^18 and 2^20,
invalid records' keys never counted, a corpus without VALID records (a digest of no entries), probe chains of ~256 keys on
one home slot and keys that wrap past the table's last slot, and 1 / 2 / 7 keys (fewer than K1h's CTAs).  The digest's
entries must be corpus_digest_model's and its fixed words the oracle report's; every report on the digest route, through
k_corpus_digest and through K1h in one launch, byte-equal to the scan's (TUNE_NO_CORPUS_DIGEST) and field-equal to the
oracle; forced grids for the smallest digests.  Corpora loaded after a digest was built (records, persisted JSON, the
generator) are reported from their own records."""
import json
import os
import random
import subprocess
import sys
from importlib import import_module

import numpy as np
import pytest

import corpus_digest_model as dm
import count_model as cm
import flagship_fixtures as ff
import k1_fixtures as kf
import test_gpu_count_route as cr
from test_gpu_candidate_corpus import check_oracle

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
W_CUSTOM = np.array([0.3, 0.1, 0.05, 0.05, 0.1, 0.1, 0.1, 0.1, 0.1])
BASES = (0, (1 << 40) + 8)


@pytest.fixture(autouse=True)
def restore(engine, apo, orc):
    engine.set_tuning(apo.TUNE_TWIN_T)
    yield
    engine.set_tuning(0)
    engine.set_weights(orc.weights())


# ------------------------------------------------------------------------------------------------ K1h
def check_counts(engine, C, T):
    """the counts the load built are count_model's pairs of the copy's index planes"""
    got = engine.debug_twin_h()
    assert got is not None
    off, pairs = got
    idx = cr.indices(engine, C, T)
    want_off, want_pairs = cm.pairs(idx, T)
    assert np.array_equal(off, want_off) and np.array_equal(pairs, want_pairs)
    return idx, off, pairs


def check_calls(engine, orc, apo, dims, C, exp=None, exp_recip=None, weights=True):
    """scores, top-K, integers and recip through K1h, K1t2 / K1t and K1q; then under weights set after the load"""
    exp = orc.score_dims_fx(dims) if exp is None else exp
    cr.routes(engine, apo, C, lambda: engine.score(C, min(3, C)), exp)
    cr.routes(engine, apo, C, lambda: engine.score(C, C, candidates=True), exp)
    cr.routes(engine, apo, C, lambda: engine.score(C, 2, recip=True), kf.fx_model(dims, recip=True) if exp_recip is None else exp_recip)
    if weights:
        engine.set_weights(W_CUSTOM)
        cr.routes(engine, apo, C, lambda: engine.score(C, C), orc.score_dims_fx(dims, w=W_CUSTOM))
        engine.set_weights(orc.weights())


def test_cap_three_batches_and_the_last_entry(engine, orc, apo):
    dims, _ = ff.cap()
    C, T = ff.CAP_C, ff.CAP_T
    engine.dims_upload(dims)
    idx, off, pairs = check_counts(engine, C, T)
    assert idx.max() == ff.TWIN_T_CAP - 1
    e, n = cm.unpack(pairs)
    last = np.flatnonzero(e == ff.TWIN_T_CAP - 1)
    assert n[last].tolist() == [1] and off[ff.CAP_SINGLE_ROW] <= last[0] < off[ff.CAP_SINGLE_ROW + 1]
    assert engine.debug_twin_t_list() is None                    # > 1/64 of the evaluations name entries >= 2^16: K1t
    check_calls(engine, orc, apo, dims, C)


def test_over_cap_builds_no_copy(engine, orc, apo):
    dims, _ = ff.cap(over=True)
    engine.dims_upload(dims)
    assert engine.debug_twin_h() is None and engine.debug_twin_t_list() is None
    check_calls(engine, orc, apo, dims, ff.CAP_C, weights=False)


def test_two_full_batches(engine, orc, apo):
    dims, _ = ff.two_batches()
    engine.dims_upload(dims)
    check_counts(engine, ff.TWO_C, ff.CAP_T)
    check_calls(engine, orc, apo, dims, ff.TWO_C, weights=False)


def test_chunk_and_slice_edges(engine, orc, apo):
    dims, _, _ = ff.chunks()
    engine.dims_upload(dims)
    _, off, pairs = check_counts(engine, ff.CH_C, ff.CH_T)
    e, _ = cm.unpack(pairs)
    row0 = e[int(off[0]):int(off[1])]
    assert (row0 >= 2 * ff.TH_CHUNK).sum() == 1 and row0.max() == 16384
    assert {31, 32, 8191, 8192, 16383} <= set(e[int(off[1]):int(off[2])].tolist())
    check_calls(engine, orc, apo, dims, ff.CH_C)


@pytest.mark.parametrize("extra", [0, 1])
def test_nnz_gate(engine, orc, apo, extra):
    dims, _ = ff.nnz_gate(extra)
    C, T = dims.shape[:2]
    engine.dims_upload(dims)
    if extra:
        assert engine.debug_twin_h() is None
    else:
        _, off, _ = check_counts(engine, C, T)
        assert 8 * int(off[C]) == C * T // 2
    check_calls(engine, orc, apo, dims, C)


def test_wide_rows_past_2_64(engine, orc, apo):
    """the exact sums as count * (the oracle's integer of each of the two evaluations); the whole tensor through the oracle
    too for the default weights"""
    rows = ff.wide_rows()[:, None, :]
    fx, _ = orc.score_dims_fx(rows)
    fr, _ = kf.fx_model(rows, recip=True)
    counts = ff.wide_counts()
    exp = ([sum(k * f for k, f in zip(r, fx)) for r in counts], [ff.WIDE_T, ff.WIDE_T])
    exp_recip = ([sum(k * f for k, f in zip(r, fr)) for r in counts], [ff.WIDE_T, ff.WIDE_T])
    assert abs(exp[0][0]) < 1 << 60 and abs(exp[0][1]) > 1 << 77
    dims = ff.wide()
    engine.dims_upload(dims)
    off, pairs = engine.debug_twin_h()
    assert off.tolist() == [0, 2, 3] and sorted(cm.unpack(pairs)[1][:2].tolist()) == sorted(ff.WIDE_SPLIT)
    assert orc.score_dims_fx(dims) == exp
    check_calls(engine, orc, apo, dims, 2, exp=exp, exp_recip=exp_recip, weights=False)
    del dims
    engine.dims_upload(np.full((1, 8, 9), np.nan, np.float32))     # free the 2.4 GB tensor for the tests after


GRID_SCRIPT = r"""
import hashlib, importlib, sys
sys.path[:0] = [sys.argv[1], sys.argv[2]]
import flagship_fixtures as ff
apo = importlib.import_module("senweaver-ide_b200")
e = apo.Engine(0)
e.set_tuning(apo.TUNE_TWIN_T)
e.dims_upload(ff.cap()[0])
off, pairs = e.debug_twin_h()
h = hashlib.sha256(off.tobytes() + pairs.tobytes())
for K in (1, 5):
    r = e.score(ff.CAP_C, K)
    h.update(repr(e.debug_partials(ff.CAP_C)).encode() + r.scores.tobytes() + r.topk.tobytes())
e.close()
print(h.hexdigest())
"""


def test_cap_forced_grids():
    """the counts' bytes and the K1h results for forced grids of 1, 2, 3 and 7 CTAs (APO_K1_GRID, read once per process)"""
    out = []
    for grid in (None, "1", "2", "3", "7"):
        env = dict(os.environ)
        env.pop("APO_K1_GRID", None)
        if grid:
            env["APO_K1_GRID"] = grid
        r = subprocess.run([sys.executable, "-c", GRID_SCRIPT, ROOT, HERE], capture_output=True, text=True, env=env, cwd=ROOT, timeout=900)
        assert r.returncode == 0, r.stderr[-2000:]
        out.append(r.stdout.split()[-1])
    assert len(set(out)) == 1, out


# ------------------------------------------------------------------------------------------------ the digest
def call(engine):
    return engine.score(cr.C, 2, corpus=True)


def digest_case(engine, apo, orc, recs, idx_base, kept):
    """load recs; the second reported call builds the digest (kept: the model's entries and the oracle's fixed words, K1h
    in one launch; else none, and the scan); every route's report bytes the scan's and its fields the oracle's"""
    engine.set_tuning(apo.TUNE_TWIN_T)
    engine.corpus_upload(recs, idx_base)
    call(engine)
    assert engine.debug_corpus_digest() is None                   # a corpus reported once builds nothing
    call(engine)
    ref = orc.report(recs, idx_base=idx_base, nthreads=16)
    got = engine.debug_corpus_digest()
    want = dm.entries(recs)
    if kept and want:
        assert got is not None
        ent, fixed = got
        assert sorted(map(tuple, ent.tolist())) == want
        assert [int(x) for x in fixed] == dm.fixed_words(ref, idx_base)
    else:
        assert got is None                                         # dropped, or kept with no entries (n = 0)
    r = call(engine)
    assert r.timing.launches == (1 if kept else 2)                # K1h + the digest pass + the tail: one launch
    scan_flags = apo.TUNE_TWIN_T | apo.TUNE_NO_CORPUS_DIGEST
    engine.set_tuning(scan_flags)
    scan = call(engine)
    engine.set_tuning(apo.TUNE_TWIN_T | apo.TUNE_NO_TWIN_H)       # K1t2, then k_corpus_digest (or the scan) with the tail
    standalone = call(engine)
    engine.set_tuning(apo.TUNE_TWIN_T)
    for x in (r, standalone):
        assert bytes(x.report) == bytes(scan.report)
        assert np.array_equal(x.scores, scan.scores) and np.array_equal(x.topk, scan.topk)
    check_oracle(apo, r.report, ref)
    return r


@pytest.fixture
def k1h_dims(engine, apo):
    engine.set_tuning(apo.TUNE_TWIN_T)
    engine.dims_upload(cr.build())
    assert engine.debug_twin_h() is not None


@pytest.mark.parametrize("idx_base", BASES)
@pytest.mark.parametrize("T", [ff.GATE_SMALL_T, ff.GATE_LARGE_T])
def test_digest_gate(engine, apo, orc, k1h_dims, T, idx_base):
    for extra in (0, 1):
        digest_case(engine, apo, orc, ff.gate(T, extra), idx_base, kept=not extra)
    if T == ff.GATE_LARGE_T:
        digest_case(engine, apo, orc, ff.gate_invalid(T), idx_base, kept=True)


def test_no_valid_record(engine, apo, orc, k1h_dims):
    r = digest_case(engine, apo, orc, ff.no_valid(), 7, kept=True)
    assert r.report.withReward == 0 and r.report.total == ff.NO_VALID_T


@pytest.mark.parametrize("idx_base", BASES)
def test_probe_chains_and_wrap(engine, apo, orc, k1h_dims, idx_base):
    recs, _, _ = ff.probe()
    digest_case(engine, apo, orc, recs, idx_base, kept=True)


@pytest.mark.parametrize("nkeys", ff.FEW)
def test_few_keys(engine, apo, orc, k1h_dims, nkeys):
    digest_case(engine, apo, orc, ff.few(nkeys), BASES[1], kept=True)


DIGEST_GRID_SCRIPT = r"""
import importlib, json, sys
sys.path[:0] = [sys.argv[1], sys.argv[2]]
import flagship_fixtures as ff
import test_gpu_count_route as cr
apo = importlib.import_module("senweaver-ide_b200")
e = apo.Engine(0)
e.set_tuning(apo.TUNE_TWIN_T)
e.dims_upload(cr.build())
out = []
for recs in [ff.no_valid()] + [ff.few(k) for k in ff.FEW]:
    e.corpus_upload(recs, 11)
    for _ in range(3):
        r = e.score(cr.C, 2, corpus=True)
    out.append({"launches": int(r.timing.launches), "report": bytes(r.report).hex(), "scores": r.scores.tolist()})
e.close()
print(json.dumps(out))
"""


def test_smallest_digests_forced_grids(apo, orc):
    """no entries and 1 / 2 / 7 entries through K1h at 1, 2, 3 and 7 CTAs: one launch, the same report and scores at every
    grid, the oracle's report"""
    refs = [orc.report(recs, idx_base=11, nthreads=16) for recs in [ff.no_valid()] + [ff.few(k) for k in ff.FEW]]
    first = None
    for g in (1, 2, 3, 7):
        p = subprocess.run([sys.executable, "-c", DIGEST_GRID_SCRIPT, ROOT, HERE], env=dict(os.environ, APO_K1_GRID=str(g)),
                           capture_output=True, text=True, timeout=900)
        assert p.returncode == 0, p.stderr[-3000:]
        out = json.loads(p.stdout.strip().splitlines()[-1])
        assert [o["launches"] for o in out] == [1] * len(refs), g
        for o, ref in zip(out, refs):
            check_oracle(apo, apo.engine.CorpusReport.from_buffer_copy(bytes.fromhex(o["report"])), ref)
        assert first is None or out == first, g
        first = out


def test_reloads_never_use_a_stale_digest(engine, apo, orc, k1h_dims):
    """after each digest is built, a smaller corpus (records, persisted JSON) and a generated one report their own records"""
    def built():
        engine.corpus_upload(ff.few(7), 0)
        call(engine)
        call(engine)
        assert call(engine).timing.launches == 1

    built()
    recs = orc.gen_records(0x5EEDF107, orc.STREAM_CORPUS, 0, 1, 0, 300_001, 300).reshape(-1)
    engine.corpus_upload(recs, 3)
    for _ in range(3):
        r = call(engine)
        assert engine.debug_corpus_digest() is None
    check_oracle(apo, r.report, orc.report(recs, idx_base=3, nthreads=16))

    built()
    svc = import_module("test_gpu_services")
    store = {}
    tc = import_module("senweaver-ide_b200.trace_collector").TraceCollectorService(engine, storageService=store)
    svc.drive(tc, random.Random(0x5EEDF106), n_threads=200)
    tc._dirty = True
    tc._saveToStorage()
    n = engine.corpus_upload_json(store["senweaver.traceCollector.data"])
    want = tc.corpus_records(tc.getAllTraces())
    assert n == len(want)
    for _ in range(3):
        r = call(engine)
        assert engine.debug_corpus_digest() is None
    check_oracle(apo, r.report, orc.report(want, nthreads=16))

    built()
    seed, T = 0x5EEDF108, (1 << 20) + 11                           # generated, large enough for a digest of its own
    engine.corpus_generate(seed, 0, T, 300)
    ref = orc.report_generated(seed, 0, T)
    for i in range(3):
        r = call(engine)
        check_oracle(apo, r.report, ref)
    assert r.timing.launches == 1 and engine.debug_corpus_digest() is not None
