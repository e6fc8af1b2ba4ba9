"""Whole rows of the Form T copy scored from its per-row dictionary counts (-m gpu, K1h: k_reward9th).  Every result must
equal the oracle's integers (the numpy model for recip) and those of the same engine with TUNE_NO_TWIN_H set after the load
(K1t2 on the slot plane) and TUNE_NO_TWIN_T (K1q on the Form W copy): integers, counts, scores, top-K, corpus report and
per-candidate breakdown.  The counts the load built must be the ones tests/count_model.py derives from the copy's index
planes (resident Form T of the same tensor builds the same dictionary)."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

import count_model as cm
import k1_fixtures as kf
import test_gpu_twin_t_list as tl
from test_gpu_dims_twin import same

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
C, T = 13, 100_003                                  # C prime, T ragged (T - 3 on the 8-grid)
NULL_ROW, ONE_ROW, RARE_ROW = 2, 5, 11
W_CUSTOM = np.array([0.3, 0.1, 0.05, 0.05, 0.1, 0.1, 0.1, 0.1, 0.1])


@pytest.fixture(autouse=True)
def forced(engine, apo):
    engine.set_tuning(apo.TUNE_TWIN_T)
    yield
    engine.set_tuning(0)


@functools.lru_cache(maxsize=1)
def build():
    """[C][T] dims: a skewed head of 300 evaluations, one all-null row, one row of a single evaluation repeated T times, and
    70 000 rare evaluations seen once (dictionary entries 2^16 and up, the exceptions) filling most of one row"""
    rng = np.random.default_rng(0x5EED7180)
    pool = tl.distinct(0x5EED7180, 300 + 70_000, tl.zero_weight_rows())
    head, rare = pool[:300], pool[300:]
    d = head[np.minimum(rng.geometric(1 / 40, (C, T)) - 1, 299)]
    d[NULL_ROW] = np.nan
    d[ONE_ROW] = head[7]
    d[RARE_ROW, :70_000] = rare
    return d


def indices(engine, Cn, Tn):
    engine.dims_tuples()
    out = np.empty((Cn, Tn), np.int64)
    for c in range(Cn):
        lo, hi = engine.tuples_download(c, 0, Tn)
        out[c] = lo.astype(np.int64) | (hi.astype(np.int64) << 16)
    return out


def routes(engine, apo, Cn, call, want, corpus=False):
    """call() under the default tuning (K1h on whole rows), TUNE_NO_TWIN_H (K1t2) and TUNE_NO_TWIN_T (K1q): the same
    integers (`want` unless None) and results"""
    out = []
    try:
        for flags in (0, apo.TUNE_NO_TWIN_H, apo.TUNE_NO_TWIN_T):
            engine.set_tuning(apo.TUNE_TWIN_T | flags)
            call()
            r = call()
            out.append((r, engine.debug_partials(Cn)))
    finally:
        engine.set_tuning(apo.TUNE_TWIN_T)
    (r0, p0) = out[0]
    if want is not None:
        assert p0 == want
    for r, p in out[1:]:
        assert p == p0 and same(r, r0)
        if corpus:
            assert memoryview(r.report).tobytes() == memoryview(r0.report).tobytes()
    return r0


def test_layout_matches_the_model(engine, orc):
    dims = build()
    engine.dims_upload(dims)
    got = engine.debug_twin_h()
    assert got is not None
    off, pairs = got
    idx = indices(engine, C, T)
    assert idx.max() >= 65536 and np.all(idx[ONE_ROW] == idx[ONE_ROW, 0])
    want_off, want_pairs = cm.pairs(idx, T)
    assert np.array_equal(off, want_off) and np.array_equal(pairs, want_pairs)
    assert off[ONE_ROW + 1] - off[ONE_ROW] == 1 and off[NULL_ROW + 1] - off[NULL_ROW] == 1


def test_calls_against_oracle(engine, orc, apo):
    dims = build()
    engine.dims_upload(dims)
    recs = orc.gen_records(0x5EED7181, orc.STREAM_CORPUS, 0, 1, 0, 20_000, 300, 8).reshape(-1)
    engine.corpus_upload(recs)
    exp = orc.score_dims_fx(dims)
    r = routes(engine, apo, C, lambda: engine.score(C, 3, corpus=True), exp, corpus=True)
    assert r.timing.launches == 2 and r.report.bad == orc.report(recs).bad
    routes(engine, apo, C, lambda: engine.score(C, 2, count=T), exp)             # the whole row as an explicit count
    routes(engine, apo, C, lambda: engine.score(C, 2, candidates=True), exp)
    for recip in (True, False):
        routes(engine, apo, C, lambda: engine.score(C, C, recip=recip), kf.fx_model(dims, recip=True) if recip else exp)
    for first, count in ((0, T - 3), (8, 0), (4096, 50_000)):                      # off the whole row: K1t2 on every setting
        end = first + count if count else T
        routes(engine, apo, C, lambda: engine.score(C, 1, first=first, count=count), orc.score_dims_fx(dims[:, first:end]))
    for K in (1, 6, C):
        routes(engine, apo, C, lambda: engine.score(C, K), exp)


def test_weights_set_after_the_load(engine, orc, apo):
    dims = build()
    engine.dims_upload(dims)
    try:
        for w in (tl.W_ZERO, W_CUSTOM, orc.weights()):
            engine.set_weights(w)
            routes(engine, apo, C, lambda: engine.score(C, C), orc.score_dims_fx(dims, w=w))
            routes(engine, apo, C, lambda: engine.score(C, 2, recip=True), kf.fx_model(dims, w=w, recip=True))
    finally:
        engine.set_weights(orc.weights())


def test_sessions_with_candidate_offsets(engine, orc, apo):
    dims = build()
    engine.dims_upload(dims)
    sums, counts = orc.score_dims_fx(dims)

    def session(cand=False):
        engine.score_begin(2 * C + 1)
        engine.score_accumulate(1, candidates=cand)                               # whole rows: K1h
        engine.score_accumulate(C + 1, count=T - 3, candidates=cand)              # K1t2 ...
        engine.score_accumulate(C + 1, first=T - 3, candidates=cand)              # ... and the rest through K1
        return engine.score_finish(2 * C + 1, 4, candidates=cand)

    want = ([0] + list(sums) * 2, [0] + list(counts) * 2)
    routes(engine, apo, 2 * C + 1, session, want)
    routes(engine, apo, 2 * C + 1, lambda: session(True), want)


def test_loads_and_the_gate(engine, orc, apo):
    dims = build()
    exp = orc.score_dims_fx(dims)
    engine.set_tuning(apo.TUNE_TWIN_T | apo.TUNE_NO_TWIN_H)                         # a load with the flag builds none
    engine.dims_upload(dims)
    assert engine.debug_twin_h() is None and engine.debug_twin_t_list() is not None
    engine.set_tuning(apo.TUNE_TWIN_T)
    engine.score(C, 2)
    assert engine.debug_partials(C) == exp
    engine.dims_upload(dims)
    first = engine.debug_twin_h()
    assert first is not None
    # a later load replaces the counts: ~5000 distinct evaluations in rows of 30 000, more pairs than the gate lets through;
    # the copy is still read, through K1t2 and the stand-alone tail (the Form W copy would take one launch).  No profiler
    # record here: a process's later records lose their kernels once its first profiler session lies tens of seconds back
    pool = tl.distinct(0x5EED7182, 5000, tl.zero_weight_rows())
    small = pool[np.random.default_rng(0x5EED7182).integers(0, 5000, (3, 30_000))]
    engine.dims_upload(small)
    assert engine.debug_twin_h() is None
    assert engine.score(3, 2).timing.launches == 2
    routes(engine, apo, 3, lambda: engine.score(3, 2), orc.score_dims_fx(small))
    engine.dims_upload(dims)
    again = engine.debug_twin_h()
    assert np.array_equal(again[0], first[0]) and np.array_equal(again[1], first[1])
    engine.dims_compact()                                                          # the copy goes, and the counts with it
    assert engine.debug_twin_h() is None


def flagship_rows(free, Tf, cap=256):
    """rows of Tf evaluations whose load keeps the Form W and Form T copies and the counts in `free` bytes.  The load's peak
    is the fp32 tensor (36 B per evaluation) + the Form Q planes the Form W words are packed from (14 B) + the words (8 B), with
    4 GiB left free beside them (kTwinHeadroom; the Form T copy, its lists and the counts come after the planes are freed and
    need less); 1 GiB more for the engine's own buffers and the corpus"""
    return min(cap, max(0, (free - (5 << 30)) // (58 * Tf)))


def test_flagship_seed(apo):
    """the benchmark's tensor (seed 0x5EED0003, 5 M evaluations per row) on an engine of its own (the tensor goes with it):
    counts held, the first and last rows as the model, every route equal.  All 256 rows on an otherwise empty 80 GB device;
    when other engines of the process hold device memory, as many of its rows as the copies' memory rules let the load keep
    (the generator gives every row the same evaluations at any row count)"""
    import torch
    seed, Tf = 0x5EED0003, 5_000_000
    Cf = flagship_rows(torch.cuda.mem_get_info()[0], Tf)
    if Cf < 32:
        pytest.skip(f"{torch.cuda.mem_get_info()[0] >> 30} GiB free: too little for 32 rows with their copies")
    e = apo.Engine(0)
    try:
        e.dims_generate(seed, 0, Cf, 0, Tf, 300)
        off, pairs = e.debug_twin_h()
        assert 8 * len(pairs) * 2 <= Cf * Tf
        e.corpus_generate(seed, 0, Tf, 300)
        routes(e, apo, Cf, lambda: e.score(Cf, Cf // 4, corpus=True), None, corpus=True)   # K as bench.py
        routes(e, apo, Cf, lambda: e.score(Cf, Cf // 4, recip=True), None)
        e.dims_tuples()
        for c in (0, Cf - 1):
            lo, hi = e.tuples_download(c, 0, Tf)
            _, p = cm.pairs((lo.astype(np.int64) | (hi.astype(np.int64) << 16))[None], Tf)
            assert np.array_equal(pairs[int(off[c]):int(off[c + 1])], p)
    finally:
        e.close()


GRID_SCRIPT = r"""
import hashlib, importlib, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {here!r})
import test_gpu_count_route as t
apo = importlib.import_module("senweaver-ide_b200")
e = apo.Engine(0)
e.set_tuning(apo.TUNE_TWIN_T)
e.dims_upload(t.build())
off, pairs = e.debug_twin_h()
h = hashlib.sha256(off.tobytes() + pairs.tobytes())
for first, count in ((0, 0), (0, t.T)):
    e.score(t.C, 3, first=first, count=count)
    h.update(repr(e.debug_partials(t.C)).encode())
e.close()
print(h.hexdigest())
"""


def test_grid_independence():
    """the counts' bytes and the integers for forced grids of 1, 2, 3 and 7 CTAs (APO_K1_GRID, read once per process)"""
    script = GRID_SCRIPT.format(root=ROOT, here=HERE)
    out = []
    for grid in (None, "1", "2", "3", "7"):
        env = dict(os.environ)
        env.pop("APO_K1_GRID", None)
        if grid:
            env["APO_K1_GRID"] = grid
        r = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, env=env, cwd=ROOT, timeout=900)
        assert r.returncode == 0, r.stderr[-2000:]
        out.append(r.stdout.split()[-1])
    assert len(set(out)) == 1, out
