"""The corpus scan and the per-candidate passes past their flush points, on the H100.

ScanAcc (csrc/apo_corpus.cuh) packs tallies, byMode, the six pattern counts and the per-dimension census into small bit
fields (the narrowest, d6, is 9 bits); they are right only because every host flushes before a lane has seen K2_CHUNK = 256
records.  The first three examples of each pattern, and the breakdown's badExamples, are merged from many warps, CTAs and
windows.  Here corpora large enough that every host flushes several times mid-range -- saturating ones (every record the
same: every lane fills the same fields to the cadence) with a closed-form report, and planted ones whose earliest hits sit
late, in crowded groups and on both sides of block, flush and window boundaries (tests/corpus_fixtures.py) -- run through
every host and are compared with the CPU oracle, and with the closed form with no tolerance:

- 36 M records (1.15 GB): the fused corpus warp of K1 / K1q / K1r (Form D, Q, R, R16) does ~34 rounds per lane, each
  k_detect6_tiles CTA ~133 tiles (two mid-CTA flushes), the grid-stride k_detect6 three rounds per lane (a subprocess with
  APO_K2_GRIDSTRIDE=1, which is read once per process); idx_base 0 and 2^40 + 8
- 15 x 5 M Form R16 (and 8 x 5 M Form R): every k_cand_corpus warp runs ~35 tiles (flush every 8), resident, streamed
  through 256 MB windows, in sessions whose windows arrive in reverse order, in candidate chunks
- k_cand_breakdown: rows whose only 'bad' evaluations are few and late, through every loader, across a window boundary and
  in reversed sessions, bit for bit against oracle/candidates.py"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import corpus_fixtures as cf
from test_gpu_candidate_corpus import check_oracle, corpus_report_of
from test_gpu_candidates import eng_list, orc_rep

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
BIG_T = 36_000_000
BIG_BASE = (1 << 40) + 8
SAT = ((0, 2, 4), 2)                    # saturating corpus: patterns P1, P3, P5 in mode 2 (agent thresholds)


@pytest.fixture(scope="module")
def oc(orc):
    from oracle import candidates
    candidates.build()
    return candidates


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def boundary_extra(T, sm):
    """positions on both sides of the flush points of the corpus hosts at this SM count: k_detect6_tiles (2048-record tiles,
    flush every 64 tiles of a CTA), the fused warp (stride sm x 32, a round = 256 records per lane) and the grid-stride kernel
    (stride 2 sm x 256); the assertions never depend on them, the oracle is the reference"""
    tiles = (T + 2047) // 2048
    pos = []
    for b in (0, sm // 2, sm - 1):
        lo = tiles * b // sm
        for k in (64, 128):
            pos += [(lo + k) * 2048 - 1, (lo + k) * 2048]
    for stride in (sm * 32, 2 * sm * 256):
        for r in (1, 2):
            t = r * 256 * stride + stride - 1
            pos += [t - stride, t]
    return pos


def big_corpus(kind, sm, idx_base):
    if kind == "saturating":
        return cf.saturating(BIG_T, *SAT), None
    recs, _, want = cf.planted(BIG_T, extra={5: boundary_extra(BIG_T, sm)}, idx_base=idx_base)
    return recs, want


def small_evals(orc, apo):
    dims = orc.gen_dims(0x5EED0C31, 0, 2, 0, 4096, 300, 2)
    roll = orc.gen_records(0x5EED0C31, orc.STREAM_ROLLOUT, 0, 2, 0, 4096, 300, 2)
    return dims, roll, apo.pack16(roll)


def check_corpus(apo, orc, rep, recs, kind, idx_base, want, ref):
    if kind == "saturating":
        # T equal values summed in sequential binary64 drift (1.3e-12 at 36 M): the oracle's integers, the exact closed form
        check_oracle_ints(rep, ref)
        cf.check_closed_form(rep, cf.closed_form(len(recs), *SAT, idx_base=idx_base))
    else:
        check_oracle(apo, rep, ref)
        cf.check_designed(rep, want)


def check_oracle_ints(rep, ref):
    assert (rep.total, rep.good, rep.bad, rep.none, rep.withReward) == (ref.total, ref.good, ref.bad, ref.none, ref.withReward)
    assert all(list(rep.byMode[m]) == list(ref.byMode[m]) for m in range(5))
    assert [rep.dim[i].count for i in range(9)] == [ref.dim[i].count for i in range(9)]
    for p in range(6):
        assert (rep.pat[p].count, rep.pat[p].flag, list(rep.pat[p].examples)) == (ref.pat[p].count, ref.pat[p].flag, list(ref.pat[p].examples))
    assert (rep.toolCalls, rep.toolSucc, rep.toolFail) == (ref.toolCalls, ref.toolSucc, ref.toolFail)


@pytest.mark.parametrize("kind,idx_base", [("saturating", BIG_BASE), ("planted", 0), ("planted", BIG_BASE), ("saturating", 0)])
def test_36M_corpus_through_every_scan_host(engine, orc, apo, sm_count, kind, idx_base):
    recs, want = big_corpus(kind, sm_count, idx_base)
    ref = orc.report(recs, idx_base=idx_base, nthreads=16)
    reps = every_scan_host(engine, orc, apo, recs, idx_base)
    first = reps["K1"]
    check_corpus(apo, orc, apo.engine.CorpusReport.from_buffer_copy(first), recs, kind, idx_base, want, ref)
    assert all(v == first for v in reps.values()), [k for k, v in reps.items() if v != first]


def every_scan_host(engine, orc, apo, recs, idx_base):
    """{host: report bytes} of the corpus `recs`: the corpus warp of K1 / K1q / K1r / K1r16 in the scoring launch,
    k_detect6_tiles, and a session"""
    engine.corpus_upload(recs, idx_base)
    dims, roll, roll16 = small_evals(orc, apo)
    reps = {}
    try:
        engine.set_tuning(apo.TUNE_FORCE_FUSE)          # the corpus warp inside the scoring launch
        for name, load, src in (("K1", lambda: engine.dims_upload(dims), apo.SRC_DIMS),
                                ("K1q", lambda: engine.dims_upload_compact(dims), apo.SRC_DIMS),
                                ("K1r", lambda: engine.rollouts_upload(roll), apo.SRC_ROLLOUTS),
                                ("K1r16", lambda: engine.rollouts16_upload(roll16), apo.SRC_ROLLOUTS)):
            load()
            r = engine.score(2, 1, source=src, corpus=True)
            assert r.timing.launches == 1, name
            reps[name] = bytes(r.report)
        engine.set_tuning(apo.TUNE_NO_FUSE)             # stand-alone k_detect6_tiles (+ fused finalisation)
        engine.dims_upload(dims)
        r = engine.score(2, 1, corpus=True)
        assert r.timing.launches == 2
        reps["tiles"] = bytes(r.report)
    finally:
        engine.set_tuning(0)
    engine.score_begin(2)
    engine.score_accumulate(0)
    reps["session"] = bytes(engine.score_finish(2, 1, corpus=True).report)
    return reps


GRIDSTRIDE_SCRIPT = r"""
import importlib, json, sys
sys.path[:0] = [sys.argv[1], sys.argv[2]]
import oracle
from test_gpu_corpus_flush import big_corpus
apo = importlib.import_module("senweaver-ide_b200")
e = apo.Engine(0)
out = []
e.dims_upload(oracle.gen_dims(0x5EED0C31, 0, 2, 0, 4096, 300, 2))
e.set_tuning(apo.TUNE_NO_FUSE)
for kind, base in json.loads(sys.argv[3]):
    e.corpus_upload(big_corpus(kind, int(sys.argv[4]), base)[0], base)
    r = e.score(2, 1, corpus=True)
    out.append(bytes(r.report).hex())
e.close()
print(json.dumps(out))
"""


def test_36M_corpus_grid_stride_kernel(engine, orc, apo, sm_count):
    """k_detect6 (grid-stride, 2 x sm CTAs x 256 lanes: three rounds per lane at 36 M) gives the report of k_detect6_tiles"""
    cases = [("saturating", BIG_BASE), ("planted", 0)]
    env = dict(os.environ, APO_K2_GRIDSTRIDE="1")
    p = subprocess.run([sys.executable, "-c", GRIDSTRIDE_SCRIPT, ROOT, HERE, json.dumps(cases), str(sm_count)], env=env,
                       capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-3000:]
    got = json.loads(p.stdout.strip().splitlines()[-1])
    dims, _, _ = small_evals(orc, apo)
    engine.dims_upload(dims)
    for (kind, base), hexrep in zip(cases, got):
        recs, want = big_corpus(kind, sm_count, base)
        engine.corpus_upload(recs, base)
        try:
            engine.set_tuning(apo.TUNE_NO_FUSE)
            tiles = bytes(engine.score(2, 1, corpus=True).report)
        finally:
            engine.set_tuning(0)
        assert bytes.fromhex(hexrep) == tiles, kind
        rep = apo.engine.CorpusReport.from_buffer_copy(bytes.fromhex(hexrep))
        if kind == "saturating":
            cf.check_closed_form(rep, cf.closed_form(BIG_T, *SAT, idx_base=base))
        else:
            cf.check_designed(rep, want)


@pytest.mark.parametrize("T", [8000, 8191, 3])
def test_small_corpus_grid_stride_kernel(engine, orc, apo, T):
    dims, _, _ = small_evals(orc, apo)
    engine.dims_upload(dims)
    for kind, base in (("saturating", BIG_BASE), ("planted", 12)):
        if kind == "saturating":
            recs = cf.saturating(T, *SAT)
        else:
            recs, _, want = cf.planted(T, idx_base=base)
        engine.corpus_upload(recs, base)
        try:
            engine.set_tuning(apo.TUNE_NO_FUSE)
            r = engine.score(2, 1, corpus=True)
        finally:
            engine.set_tuning(0)
        check_oracle(apo, r.report, orc.report(recs, idx_base=base))
        if kind == "saturating":
            cf.check_closed_form(r.report, cf.closed_form(T, *SAT, idx_base=base))
        else:
            cf.check_designed(r.report, want)


# ------------------------------------------------------------------------------------------------ k_cand_corpus
CC_C, CC_T = 15, 5_000_000          # 15 rows: no warp of k_cand_corpus (132 x k x 8 of them) starts exactly at a row


def host_window(C, row, T, tile=2560):
    """the record window of apo_score_host_records: 256 MB / (C x row), a multiple of the K1 tile (csrc/apo_abi.cu)"""
    tc = (256 << 20) // (C * row) // tile * tile
    return min(max(tc, tile), (T + tile - 1) // tile * tile)


def cand_rows16(sm):
    """15 rows of 5 M Form R16: planted rows (scenarios rotated and shifted per row; pairs on both sides of the first window
    boundary of the streamed call with the earliest hit of one pattern in the second window; pairs on both sides of the warp
    and flush boundaries of k_cand_corpus for 1-4 CTAs per SM) and, as rows 5 and 11, saturating rows"""
    Tc = host_window(CC_C, 16, CC_T)
    tpc = (CC_T + 1023) // 1024
    total = tpc * CC_C
    rows = np.empty((CC_C, CC_T), cf.oracle.RECORD16_DTYPE)
    for c in range(CC_C):
        if c in (5, 11):
            rows[c] = cf.saturating(CC_T, (1, 3, 5) if c == 5 else tuple(range(6)), mode=2 if c == 5 else 1, row=16)
            continue
        extra = [Tc + 5 + c, 2 * Tc - 1, 2 * Tc]
        for per_sm in (1, 2, 3, 4):
            nw = sm * per_sm * 8
            gw = (c * tpc + tpc // 2) * nw // total              # a warp inside this row, its first tile and its flushes
            lo = -(-total * gw // nw) - c * tpc
            for k in (0, 8, 16):
                extra += [(lo + k) * 1024 - 1, (lo + k) * 1024]
        rows[c] = cf.planted(CC_T, kinds=[(p + c) % 6 for p in range(6)], shift=97 * c, extra={c % 6: extra}, row=16)[0]
    return rows


@pytest.fixture(scope="module")
def cc_rows(orc, sm_count):
    p16 = cand_rows16(sm_count)
    refs = [orc.report(orc.unpack16(p16[c]), nthreads=16) for c in range(CC_C)]
    return p16, refs


def check_cc(engine, apo, orc, reports, p16, refs):
    """each report byte-equal to the engine's corpus report of its row, field-equal to the oracle, and the closed form for
    the saturating rows (whose binary64 sums the oracle's sequential summation cannot give to 1e-12)"""
    for c in range(len(reports)):
        assert bytes(reports[c]) == bytes(corpus_report_of(engine, apo, orc.unpack16(p16[c]))), c
        if c in (5, 11):
            check_oracle_ints(reports[c], refs[c])
            cf.check_closed_form(reports[c], cf.closed_form(CC_T, (1, 3, 5) if c == 5 else tuple(range(6)), 2 if c == 5 else 1))
        else:
            check_oracle(apo, reports[c], refs[c])


def test_cand_corpus_16x5M_resident_streamed_r16_and_r(engine, orc, apo, cc_rows):
    p16, refs = cc_rows
    engine.rollouts16_upload(p16)
    one = engine.score(CC_C, 4, source=apo.SRC_ROLLOUTS, candidate_corpus=True).candidate_corpus
    one_b = [bytes(r) for r in one]
    check_cc(engine, apo, orc, one, p16, refs)
    # streamed: five 256 MB windows per call, hits on both sides of the first boundary
    assert host_window(CC_C, 16, CC_T) < CC_T // 4
    streamed = engine.score_host_records(p16, 4, candidate_corpus=True).candidate_corpus
    assert [bytes(r) for r in streamed] == one_b
    # Form R: the same records, eight rows at a time (32 B each)
    for c0 in (0, 8):
        r32 = orc.unpack16(p16[c0:c0 + 8])
        engine.rollouts_upload(r32)
        res = engine.score(len(r32), 2, source=apo.SRC_ROLLOUTS, candidate_corpus=True)
        assert [bytes(r) for r in res.candidate_corpus] == one_b[c0:c0 + 8]
        if c0 == 0:
            assert [bytes(r) for r in engine.score_host_records(r32, 2, candidate_corpus=True).candidate_corpus] == one_b[:8]
        del r32


def test_cand_corpus_reversed_windows_and_candidate_chunks(engine, orc, apo, cc_rows):
    p16, refs = cc_rows
    engine.rollouts16_upload(p16)
    one = [bytes(r) for r in engine.score(CC_C, 4, source=apo.SRC_ROLLOUTS, candidate_corpus=True).candidate_corpus]
    # later records first: every window's hits must be displaced by the earlier windows' hits that arrive after them
    cuts = [0, 1_048_576, 2_000_000, 2_000_004, 4_999_000, CC_T]
    engine.score_begin(CC_C)
    for a, b in reversed(list(zip(cuts, cuts[1:]))):
        engine.score_accumulate(0, source=apo.SRC_ROLLOUTS, first=a, count=b - a, candidate_corpus=True)
    assert [bytes(r) for r in engine.score_finish(CC_C, 4, candidate_corpus=True).candidate_corpus] == one
    # the second half of the rows alone, as one window: examples are absolute positions
    engine.score_begin(CC_C)
    engine.score_accumulate(0, source=apo.SRC_ROLLOUTS, first=2_500_000, count=0, candidate_corpus=True)
    half = engine.score_finish(CC_C, 4, candidate_corpus=True).candidate_corpus
    for c in (0, 3, 5, 9):
        check_oracle(apo, half[c], orc.report(orc.unpack16(p16[c, 2_500_000:]), idx_base=2_500_000, nthreads=16))
    # candidate chunks in reverse order, each in reversed windows
    engine.score_begin(CC_C)
    for c0 in (8, 0):
        engine.rollouts16_upload(p16[c0:c0 + 8])
        engine.score_accumulate(c0, source=apo.SRC_ROLLOUTS, first=3_000_000, count=0, candidate_corpus=True)
        engine.score_accumulate(c0, source=apo.SRC_ROLLOUTS, first=0, count=3_000_000, candidate_corpus=True)
    assert [bytes(r) for r in engine.score_finish(CC_C, 4, candidate_corpus=True).candidate_corpus] == one


# ------------------------------------------------------------------------------------------------ k_cand_breakdown
BD_C, BD_T = 5, 2_500_000             # 5 rows: no warp of k_cand_breakdown (132 x k x 8 of them) starts exactly at a row


def bd_positions(Tc):
    """sparse late 'bad' positions per row (corpus_fixtures.sparse_bad_positions): row 0 ends in a 'bad' evaluation and row 1
    holds only two, so a warp that carried row 0's first positions into row 1 would show; row 2 gets its earliest 'bad'
    evaluation just inside the second window of the streaming calls (Tc), row 3 a pair on both sides of that boundary"""
    pos = cf.sparse_bad_positions(BD_C, BD_T)
    pos[2] = sorted(set(pos[2]) | {Tc + 9, Tc + 10})
    pos[3] = sorted(set(pos[3]) | {Tc - 1, Tc})
    assert pos[0][-1] == BD_T - 1 and len(pos[1]) == 2
    return pos


def test_breakdown_sparse_late_bad_dims_every_loader(engine, orc, apo, oc):
    Tc = host_window(BD_C, 36, BD_T)
    assert Tc < BD_T
    pos = bd_positions(Tc)
    dims = cf.sparse_bad_dims(orc.gen_dims(0x5EED0C32, 0, BD_C, 0, BD_T, 300, 16), pos)
    ref = [orc_rep(d) for d in oc.cand_dims(dims)]
    for c, d in enumerate(ref):
        assert d["bad"] == len(pos[c]) and d["badExamples"] == (pos[c][:3] + [-1] * 3)[:3]
    engine.dims_upload(dims)
    assert eng_list(engine.score(BD_C, 2, candidates=True).candidates) == ref                         # Form D resident
    assert eng_list(engine.score_host(dims, 2, candidates=True).candidates) == ref                    # Form D streamed, 2 windows
    engine.score_begin(BD_C)                                                                          # reversed windows
    engine.score_accumulate(0, first=1_250_000, count=0, candidates=True)
    engine.score_accumulate(0, first=0, count=1_250_000, candidates=True)
    assert eng_list(engine.score_finish(BD_C, 2, candidates=True).candidates) == ref
    engine.dims_upload_compact(dims)
    assert eng_list(engine.score(BD_C, 2, candidates=True).candidates) == ref                         # Form Q resident
    engine.score_begin(BD_C)
    engine.score_accumulate(0, first=2_000_000, count=0, candidates=True)
    engine.score_accumulate(0, first=0, count=2_000_000, candidates=True)
    assert eng_list(engine.score_finish(BD_C, 2, candidates=True).candidates) == ref
    q8, d2, li, book = apo.compact_encode_host(dims, nthreads=16)
    assert eng_list(engine.score_host_compact(q8, d2, li, book, 2, candidates=True).candidates) == ref
    del q8, d2, li
    pc, pd, pbook, d2book = apo.packed_encode_host(dims, nthreads=16)
    del dims
    assert eng_list(engine.score_host_packed(pc, pd, pbook, d2book, 2, candidates=True).candidates) == ref   # Form P streamed
    tl, th, tbook = apo.tuple_encode_host(pc, pd, nthreads=16)
    del pc, pd
    assert eng_list(engine.score_host_tuples(tl, th, tbook, pbook, d2book, 2, candidates=True).candidates) == ref
    engine.tuples_upload(tl, th, tbook, pbook, d2book)
    assert eng_list(engine.score(BD_C, 2, source=apo.SRC_TUPLES, candidates=True).candidates) == ref       # Form T resident
    engine.score_begin(BD_C)
    engine.score_accumulate(0, source=apo.SRC_TUPLES, first=1_000_000, count=0, candidates=True)
    engine.score_accumulate(0, source=apo.SRC_TUPLES, first=0, count=1_000_000, candidates=True)
    assert eng_list(engine.score_finish(BD_C, 2, candidates=True).candidates) == ref


def test_breakdown_sparse_late_bad_records(engine, orc, apo, oc):
    Tc = host_window(BD_C, 32, BD_T)
    assert Tc < BD_T
    pos = bd_positions(Tc)
    idx = np.stack([cf.background_index(BD_T)] * BD_C)
    idx[(idx >= 10) & (idx < 15)] -= 10                          # no background 'bad' record: only the planted ones
    for c, q in enumerate(pos):
        idx[c, q] = 10 + c
    for row in (32, 16):
        recs = cf.table(row)[idx]
        rows32 = recs if row == 32 else orc.unpack16(recs)
        ref = [orc_rep(d) for d in oc.cand_records(rows32)]
        for c, d in enumerate(ref):
            assert d["bad"] == len(pos[c]) and d["badExamples"] == (pos[c][:3] + [-1] * 3)[:3]
        if row == 32:
            engine.rollouts_upload(recs)
        else:
            engine.rollouts16_upload(recs)
        assert eng_list(engine.score(BD_C, 2, source=apo.SRC_ROLLOUTS, candidates=True).candidates) == ref
        assert eng_list(engine.score_host_records(recs, 2, candidates=True).candidates) == ref
        engine.score_begin(BD_C)
        engine.score_accumulate(0, source=apo.SRC_ROLLOUTS, first=Tc, count=0, candidates=True)
        engine.score_accumulate(0, source=apo.SRC_ROLLOUTS, first=0, count=Tc, candidates=True)
        assert eng_list(engine.score_finish(BD_C, 2, candidates=True).candidates) == ref
