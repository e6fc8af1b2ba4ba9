"""The per-candidate breakdown (k_cand_breakdown / k_cand_report, csrc/apo_cand.cu) at its edges on the H100, bit for bit
against the CPU oracle (oracle/candidates.py, itself pinned to an exact model by tests/test_cand_fixtures_cpu.py):

- every fixture of tests/cand_fixtures.py (sums past 2^64 and 2^83 that cancel across warps, binary64 and to_fx ties, the
  report thresholds, the tallies, ragged row ends) through every loader that can carry it: Form D resident (K1) and
  streamed, the Form W copy, the Form T copy with and without its exception list, Form Q resident and streamed, Form P
  streamed, Form T resident and streamed;
- windows on the 8-grid but off the 32-grid, and a session whose windows arrive in reverse order;
- forced grids of 1, 2, 3 and 7 CTAs (APO_K1_GRID, read once per process: a subprocess each) give the default grid's bytes;
- the run flush every CB_RUN_TILES = 65 536 tiles, reached at one CTA over 600 M generated evaluations of one candidate;
- the domain: a counted dimension value with |v| >= 2048 fails the call with APO_E_ARG on every source (and a session at
  apo_score_finish), leaves no breakdown behind, and the next call is exact; the same tensor without the flag scores the
  oracle's integers, and 2048 - 2^-13 is accepted.

No torch.profiler records are taken here: the routes are those pinned by test_gpu_dims_word / test_gpu_dims_tuple_copy /
test_gpu_twin_t_list under the same tuning flags."""
import json
import os
import subprocess
import sys

import pytest

import cand_fixtures as cf
from test_gpu_candidates import assert_same, eng_list, orc_rep

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
E_ARG, E_STATE = -1, -3


@pytest.fixture(scope="module")
def oc(orc):
    from oracle import candidates
    candidates.build()
    return candidates


@pytest.fixture(autouse=True)
def restore(engine, orc):
    yield
    engine.set_tuning(0)
    engine.set_weights(orc.weights())


def check(res, ref, *where):
    """every field bit for bit, and avgReward == scores[c]"""
    try:
        assert_same(res.candidates, ref, res.scores, res.counts)
    except AssertionError as e:
        raise AssertionError(f"{where}: {e}") from None


def loaders(engine, apo, dims):
    """(name, call) for every loader of the breakdown over dims; call() -> ScoreResult of a K = 1 call with the flag"""
    C = dims.shape[0]
    pc, pd, pbook, d2book = apo.packed_encode_host(dims)
    tl, th, tbook = apo.tuple_encode_host(pc, pd)
    q8, d2, li, qbook = apo.compact_encode_host(dims)

    def resident(tuning, load):
        def call(**kw):
            engine.set_tuning(tuning)
            load()
            return engine.score(C, 1, candidates=True, **kw)
        return call

    def tuples(**kw):
        engine.tuples_upload(tl, th, tbook, pbook, d2book)
        return engine.score(C, 1, source=apo.SRC_TUPLES, candidates=True, **kw)

    return [
        ("D", resident(apo.TUNE_NO_TWIN, lambda: engine.dims_upload(dims))),
        ("D host", lambda **kw: engine.score_host(dims, 1, candidates=True, **kw)),
        ("W copy", resident(0, lambda: engine.dims_upload(dims))),
        ("T copy", resident(apo.TUNE_TWIN_T, lambda: engine.dims_upload(dims))),
        ("T copy no list", resident(apo.TUNE_TWIN_T | apo.TUNE_NO_TWIN_T2, lambda: engine.dims_upload(dims))),
        ("Q", resident(0, lambda: engine.dims_upload_compact(dims))),
        ("Q host", lambda **kw: engine.score_host_compact(q8, d2, li, qbook, 1, candidates=True, **kw)),
        ("P host", lambda **kw: engine.score_host_packed(pc, pd, pbook, d2book, 1, candidates=True, **kw)),
        ("T", tuples),
        ("T host", lambda **kw: engine.score_host_tuples(tl, th, tbook, pbook, d2book, 1, candidates=True, **kw)),
    ]


def fixtures():
    yield "large_sums", cf.large_sums(), cf.W_BIG
    yield "ties", cf.ties(), cf.W_BIG
    yield "report_rules", cf.report_rules(), cf.W_BIG
    yield "tallies", cf.tallies(), cf.W_BIG
    for r in cf.SHAPE_TAILS:
        yield f"shapes_{r}", cf.shapes(r), None
    yield "many_short", cf.many_short(), None


@pytest.mark.parametrize("name", ["large_sums", "ties", "report_rules", "tallies", "shapes", "many_short"])
def test_fixtures_on_every_loader_equal_the_oracle(engine, orc, apo, oc, name):
    for fname, dims, w in fixtures():
        if not fname.startswith(name):
            continue
        w = orc.weights() if w is None else w
        engine.set_weights(w)
        ref = oc.cand_dims(dims, w=w)
        for lname, call in loaders(engine, apo, dims):
            check(call(), ref, fname, lname)


def test_windows_off_the_32_grid_and_reversed_sessions(engine, orc, apo, oc):
    dims = cf.shapes(129)
    C, T = dims.shape[:2]
    w = orc.weights()
    for lname, call in loaders(engine, apo, dims):
        if "host" in lname:
            continue                                                   # the host-streaming calls take no window
        for first, count in ((8, 1000), (40, 0), (1000, 153)):
            end = first + count if count else T
            res = call(first=first, count=count)
            assert eng_list(res.candidates) == [orc_rep(d) for d in oc.cand_dims(dims[:, first:end], w=w, idx_base=first)], (lname, first)
    ref = [orc_rep(d) for d in oc.cand_dims(dims)]
    for tuning, load, src in ((apo.TUNE_NO_TWIN, engine.dims_upload, apo.SRC_DIMS), (0, engine.dims_upload, apo.SRC_DIMS),
                              (0, engine.dims_upload_compact, apo.SRC_DIMS)):
        engine.set_tuning(tuning)
        load(dims)
        engine.score_begin(C)
        for first, count in ((808, 0), (40, 768), (8, 32), (0, 8)):
            engine.score_accumulate(0, source=src, first=first, count=count, candidates=True)
        assert eng_list(engine.score_finish(C, 1, candidates=True).candidates) == ref, tuning


GRID_SCRIPT = r"""
import json, sys
sys.path[:0] = [sys.argv[1], sys.argv[2]]
from importlib import import_module
import cand_fixtures as cf
import oracle
apo = import_module("senweaver-ide_b200")
e = apo.Engine(0)
out = {}
try:
    for name, dims, w in (("large", cf.large_sums(), cf.W_BIG), ("short", cf.many_short(), None), ("ties", cf.ties(), cf.W_BIG)):
        e.set_weights(oracle.weights() if w is None else w)
        C = dims.shape[0]
        for lname, tuning, load in (("D", apo.TUNE_NO_TWIN, e.dims_upload), ("W", 0, e.dims_upload),
                                    ("T", apo.TUNE_TWIN_T, e.dims_upload), ("Q", 0, e.dims_upload_compact)):
            e.set_tuning(tuning)
            load(dims)
            out[name + lname] = b"".join(bytes(r) for r in e.score(C, 1, candidates=True).candidates).hex()
finally:
    e.close()
print(json.dumps(out))
"""


def grid_bytes(grid):
    env = dict(os.environ)
    env.pop("APO_K1_GRID", None)
    if grid:
        env["APO_K1_GRID"] = str(grid)
    p = subprocess.run([sys.executable, "-c", GRID_SCRIPT, ROOT, HERE], env=env, capture_output=True, text=True, timeout=1200)
    assert p.returncode == 0, p.stderr[-4000:]
    return json.loads(p.stdout.strip().splitlines()[-1])


def test_forced_grids_give_the_default_bytes():
    base = grid_bytes(None)
    for grid in (1, 2, 3, 7):
        assert grid_bytes(grid) == base, grid


FLUSH_SCRIPT = r"""
import json, os, sys
sys.path[:0] = [sys.argv[1], sys.argv[2]]
from importlib import import_module
import oracle
from oracle import candidates as oc
from test_gpu_candidates import orc_rep, eng_rep
apo = import_module("senweaver-ide_b200")
seed, T = 0x5EEDCAFF, 600_000_000
ref = [orc_rep(d) for d in oc.cand_generated(seed, [0], 0, T, 300, nthreads=os.cpu_count())]
e = apo.Engine(0)
bad = []
try:
    e.dims_generate(seed, 0, 1, 0, T, 300)
    for tuning in (apo.TUNE_NO_TWIN, 0):
        e.set_tuning(tuning)
        r = e.score(1, 1, candidates=True)
        if [eng_rep(c) for c in r.candidates] != ref:
            bad.append(tuning)
finally:
    e.close()
print(json.dumps({"bad": bad, "total": ref[0]["total"], "bad_examples": ref[0]["badExamples"]}))
"""


def test_run_flush_at_one_cta_over_600M_evaluations():
    """one CTA of 8 warps over C = 1, T = 6e8: ~73 000 tiles per warp, so every warp flushes mid-row after 65 536 tiles (and
    resets its first-three 'bad' slots there); the fp32 route (K1) and the default route"""
    env = dict(os.environ, APO_K1_GRID="1")
    p = subprocess.run([sys.executable, "-c", FLUSH_SCRIPT, ROOT, HERE], env=env, capture_output=True, text=True, timeout=3000)
    assert p.returncode == 0, p.stderr[-4000:]
    out = json.loads(p.stdout.strip().splitlines()[-1])
    assert out["total"] == 600_000_000 and out["bad"] == [], out


def test_domain_refusals_on_every_source(engine, orc, apo, oc):
    ok_dims, ok_w = cf.domain(cf.BIG, "counted")
    for v, where in cf.domain_cases():
        dims, w = cf.domain(v, where)
        C = dims.shape[0]
        engine.set_weights(w)
        refused = cf.domain_refused(v, where)
        try:
            ref = oc.cand_dims(dims, w=w)
            assert not refused
        except oc.CandDomainError:
            assert refused
            ref = None
        for lname, call in loaders(engine, apo, dims):
            if refused:
                with pytest.raises(apo.ApoError) as ei:
                    call()
                assert ei.value.code == E_ARG, (v, where, lname)
                with pytest.raises(apo.ApoError) as ei:
                    engine.candidate_reports(0, C)
                assert ei.value.code == E_STATE, (v, where, lname)
            else:
                check(call(), ref, v, where, lname)
        if refused:                                                    # without the flag: the call scores the oracle's integers
            engine.set_tuning(apo.TUNE_NO_TWIN)
            engine.dims_upload(dims)
            engine.score(C, 1)
            assert engine.debug_partials(C) == orc.score_dims_fx(dims, w=w), (v, where)
            engine.set_weights(ok_w)                                   # and the next flagged call is exact
            engine.dims_upload(ok_dims)
            check(engine.score(C, 1, candidates=True), oc.cand_dims(ok_dims, w=ok_w), v, where)
            engine.set_tuning(0)


def test_a_session_refuses_at_finish_when_one_window_holds_the_value(engine, orc, apo, oc):
    dims, w = cf.domain(3000.0, "counted")                             # evaluation 37 of candidate 1
    C = dims.shape[0]
    engine.set_weights(w)
    for tuning in (apo.TUNE_NO_TWIN, 0):
        engine.set_tuning(tuning)
        engine.dims_upload(dims)
        engine.score_begin(C)
        engine.score_accumulate(0, first=0, count=32, candidates=True)
        r = engine.score_finish(C, 1, candidates=True)                 # the window without the value: exact
        assert eng_list(r.candidates) == [orc_rep(d) for d in oc.cand_dims(dims[:, :32], w=w)]
        engine.score_accumulate(0, first=32, count=0, candidates=True)
        with pytest.raises(apo.ApoError) as ei:
            engine.score_finish(C, 1, candidates=True)
        assert ei.value.code == E_ARG
        with pytest.raises(apo.ApoError) as ei:
            engine.candidate_reports(0, C)
        assert ei.value.code == E_STATE
