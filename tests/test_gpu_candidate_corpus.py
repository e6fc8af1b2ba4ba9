"""Per-candidate corpus reports (APO_SCORE_CANDIDATE_CORPUS, apo_candidate_corpus_reports) on the H100: report c is byte for
byte the engine's corpus report of candidate c's scored rollout records, and its fields equal the CPU oracle's report of that
row (compared as test_gpu_parity.check_report does) — on Form R and R16, resident and streamed from the host, in windowed
sessions and candidate chunks, at every pattern threshold, with custom and zero weights; the flag-clear path is unchanged and
every source without record fields is refused."""
import numpy as np
import pytest

from test_gpu_candidates import _bits, boundary_records
from test_gpu_parity import check_report

pytestmark = pytest.mark.gpu


def corpus_report_of(engine, apo, row, idx_base=0):
    """the engine's own corpus report (APO_SCORE_CORPUS) with `row` uploaded as the corpus"""
    engine.corpus_upload(row, idx_base)
    engine.dims_upload(np.full((1, 4, 9), np.nan, np.float32))
    return engine.score(1, 0, corpus=True).report


def check_oracle(apo, rep, ref):
    """check_report, except that a dimension whose average lies within 1e-12 of a flag threshold (-0.5, -0.3, 0) may fall on
    either side: the engine sums exactly, the oracle in sequential binary64, so such an average can round across it"""
    r = apo.engine.CorpusReport.from_buffer_copy(bytes(rep))
    for i in range(9):
        if any(abs(ref.dim[i].avg - t) < 1e-12 for t in (-0.5, -0.3, 0.0)):
            for f in ("low_flag", "low_severity", "sugg_flag", "sugg_priority"):
                setattr(r.dim[i], f, getattr(ref.dim[i], f))
    check_report(r, ref)


def assert_rows(engine, apo, orc, reports, rows, idx_base=0, w=None):
    for c, row in enumerate(rows):
        rep = corpus_report_of(engine, apo, row, idx_base)
        assert bytes(reports[c]) == bytes(rep), c
        check_oracle(apo, reports[c], orc.report(row, idx_base=idx_base, w=w))


def test_rollouts_r_r16_resident_and_streamed(engine, orc, apo):
    C, T = 4, 24_000
    recs = boundary_records(orc, C, T)
    engine.rollouts_upload(recs)
    res = engine.score(C, 2, source=apo.SRC_ROLLOUTS, candidate_corpus=True)
    assert res.candidates is None
    cc = [bytes(r) for r in res.candidate_corpus]
    streamed = engine.score_host_records(recs, 2, candidate_corpus=True)
    assert [bytes(r) for r in streamed.candidate_corpus] == cc
    assert_rows(engine, apo, orc, res.candidate_corpus, recs)
    # Form R16 (representable records: the generator's)
    gen = orc.gen_records(0x5EED0C21, orc.STREAM_ROLLOUT, 0, C, 0, 30_001, 300, 8)
    p16 = apo.pack16(gen)
    rows16 = orc.unpack16(p16)
    engine.rollouts16_upload(p16)
    res16 = engine.score(C, 2, source=apo.SRC_ROLLOUTS, candidate_corpus=True)
    assert [bytes(r) for r in engine.score_host_records(p16, 2, candidate_corpus=True).candidate_corpus] == [bytes(r) for r in res16.candidate_corpus]
    assert_rows(engine, apo, orc, res16.candidate_corpus, rows16)


def pattern_rows(orc):
    """one row per (pattern, n 'bad' hits) for n = 1..5 (minimum counts 2 / 3, severity steps at 4 and 5), plus a row whose
    records hit every predicate without a single 'bad' feedback (APO:641)"""
    T = 64
    base = np.zeros(T, orc.RECORD_DTYPE)
    base["feedback"] = 1
    base["flags"] = 0x08 | 0x02
    base["mode"] = np.arange(T) % 5
    base["userMsgs"], base["asstMsgs"], base["toolCalls"], base["toolSucc"] = 1, 1, 1, 1
    base["llmCalls"], base["tokens"], base["toolDurMs"] = 1, 500, 100.0
    base[7]["feedback"] = 2                                                     # a 'bad' record that hits no predicate

    def hit(r, p):
        if p == 0: r["flags"] |= 0x01
        elif p == 1: r["flags"] |= 0x10; r["toolFail"] = 1; r["toolSucc"] = 0
        elif p == 2: r["tokens"] = 10_001
        elif p == 3: r["llmCalls"] = 3
        elif p == 4: r["userMsgs"] = 4
        else: r["toolDurMs"] = 20_000.0

    rows, want = [], []
    for p in range(6):
        for n in range(1, 6):
            row = base.copy()
            for k in range(n):
                i = 3 + 11 * k
                row[i]["feedback"] = 2
                hit(row[i:i + 1], p)
            rows.append(row)
            want.append((p, n))
    calm = base.copy()
    calm["feedback"] = 1
    for p in range(6):
        hit(calm[10 * p:10 * p + 5], p)
    rows.append(calm)
    return np.stack(rows), want


def test_patterns_at_their_thresholds_and_the_no_bad_row(engine, orc, apo):
    rows, want = pattern_rows(orc)
    C = rows.shape[0]
    engine.rollouts_upload(rows)
    res = engine.score(C, 1, source=apo.SRC_ROLLOUTS, candidate_corpus=True)
    assert_rows(engine, apo, orc, res.candidate_corpus, rows)
    minc, sev = (2, 2, 3, 2, 2, 2), {0: lambda n: 2 if n >= 5 else 1, 1: lambda n: 2 if n >= 5 else 1, 2: lambda n: 1,
                                     3: lambda n: 2, 4: lambda n: 2 if n >= 4 else 1, 5: lambda n: 1}
    for c, (p, n) in enumerate(want):
        q = res.candidate_corpus[c].pat[p]
        assert (q.count, q.flag) == (n, int(n >= minc[p])), (p, n)
        if q.flag:
            assert q.severity == sev[p](n), (p, n)
        assert [int(x) for x in q.examples] == [3 + 11 * k for k in range(min(n, 3))] + [-1] * (3 - min(n, 3))
    calm = res.candidate_corpus[C - 1]
    assert calm.bad == 0 and all(calm.pat[p].count == 0 and calm.pat[p].flag == 0 for p in range(6))


def test_both_flags_share_fields_with_the_breakdown(engine, orc, apo):
    C, T = 5, 20_000
    recs = boundary_records(orc, C, T, seed=21)
    engine.rollouts_upload(recs)
    res = engine.score(C, 3, source=apo.SRC_ROLLOUTS, candidates=True, candidate_corpus=True)
    for c in range(C):
        b, r = res.candidates[c], res.candidate_corpus[c]
        for f in ("total", "good", "bad", "none", "withReward"):
            assert getattr(b, f) == getattr(r, f), (c, f)
        for f in ("goodRate", "rewardSum", "avgReward"):
            assert _bits(getattr(b, f)) == _bits(getattr(r, f)), (c, f)
        assert bytes(b.dim) == bytes(r.dim), c
        if res.counts[c]:
            assert _bits(r.avgReward) == _bits(res.scores[c])                 # RECIP not set: the score's own division


def test_windowed_sessions_and_candidate_chunks_equal_one_call(engine, orc, apo):
    C, T = 6, 40_000
    recs = boundary_records(orc, C, T, seed=5)
    engine.rollouts_upload(recs)
    one = [bytes(r) for r in engine.score(C, 2, source=apo.SRC_ROLLOUTS, candidate_corpus=True).candidate_corpus]
    engine.score_begin(C)
    for c0 in (0, 3):
        engine.rollouts_upload(recs[c0:c0 + 3])
        engine.score_accumulate(c0, source=apo.SRC_ROLLOUTS, first=0, count=16_000, candidate_corpus=True)
        engine.score_accumulate(c0, source=apo.SRC_ROLLOUTS, first=16_000, count=0, candidate_corpus=True)
    assert [bytes(r) for r in engine.score_finish(C, 2, candidate_corpus=True).candidate_corpus] == one
    assert [bytes(r) for r in engine.score_finish(C, 2, candidate_corpus=True).candidate_corpus] == one   # finish may be repeated
    # one window [first, first + count): absolute record positions
    engine.rollouts_upload(recs)
    first, count = 12, 10_000
    engine.score_begin(C)
    engine.score_accumulate(0, source=apo.SRC_ROLLOUTS, first=first, count=count, candidate_corpus=True)
    win = engine.score_finish(C, 1, candidate_corpus=True).candidate_corpus
    assert_rows(engine, apo, orc, win, recs[:, first:first + count], idx_base=first)
    # a mixed session refuses the reports; out-of-range requests are argument errors
    engine.score_begin(C)
    engine.score_accumulate(0, source=apo.SRC_ROLLOUTS, first=0, count=20_000, candidate_corpus=True)
    engine.score_accumulate(0, source=apo.SRC_ROLLOUTS, first=20_000, count=0)
    with pytest.raises(apo.ApoError) as ei:
        engine.score_finish(C, 2, candidate_corpus=True)
    assert ei.value.code == -3
    with pytest.raises(apo.ApoError) as ei:
        engine.candidate_corpus_reports(0, C)
    assert ei.value.code == -3
    engine.score(C, 2, source=apo.SRC_ROLLOUTS, candidate_corpus=True)
    with pytest.raises(apo.ApoError) as ei:
        engine.candidate_corpus_reports(C - 1, 2)
    assert ei.value.code == -1


def test_custom_and_zero_weights(engine, orc, apo):
    C, T = 3, 8_000
    recs = boundary_records(orc, C, T, seed=3)
    try:
        for w in (np.array([0.0, 0.3, 0.0, 0.1, 0.2, 0.0, 0.1, 0.2, 0.1]), np.array([0.0] * 8 + [1.0]), np.linspace(0.05, 0.45, 9)):
            engine.set_weights(w)
            engine.rollouts_upload(recs)
            res = engine.score(C, 2, source=apo.SRC_ROLLOUTS, candidate_corpus=True)
            assert_rows(engine, apo, orc, res.candidate_corpus, recs, w=w)
    finally:
        engine.set_weights(orc.weights())


def test_many_candidates(engine, orc, apo):
    C, T = 16384, 96
    recs = boundary_records(orc, C, T, seed=8)
    engine.rollouts_upload(recs)
    res = engine.score(C, 16, source=apo.SRC_ROLLOUTS, candidate_corpus=True)
    assert_rows(engine, apo, orc, res.candidate_corpus, recs)


def test_flag_clear_is_unchanged_and_refusals(engine, orc, apo):
    C, T = 6, 50_000
    recs = boundary_records(orc, C, T, seed=9)
    corpus = orc.gen_records(0x5EED0C22, orc.STREAM_CORPUS, 0, 1, 0, 3000, 300, 8).reshape(-1)
    engine.rollouts_upload(recs)
    engine.corpus_upload(corpus)

    def plain(**kw):
        r = engine.score(C, 3, source=apo.SRC_ROLLOUTS, corpus=True, **kw)
        return (r.scores.tobytes(), r.counts.tobytes(), r.topk.tobytes(), bytes(r.report), engine.debug_partials(C),
                r.timing.launches, r.candidate_corpus)

    before = plain()
    flagged = engine.score(C, 3, source=apo.SRC_ROLLOUTS, corpus=True, candidate_corpus=True)
    after = plain()
    assert before == after and before[-1] is None
    assert flagged.scores.tobytes() == before[0] and flagged.topk.tobytes() == before[2] and bytes(flagged.report) == before[3]
    assert flagged.timing.launches == before[5] + 2                     # the corpus pass + its report kernel
    cand_only = engine.score(C, 3, source=apo.SRC_ROLLOUTS, corpus=True, candidates=True)
    with pytest.raises(apo.ApoError) as ei:                             # the last call did not set the flag
        engine.candidate_corpus_reports(0, C)
    assert ei.value.code == -3
    both = engine.score(C, 3, source=apo.SRC_ROLLOUTS, corpus=True, candidates=True, candidate_corpus=True)
    assert both.timing.launches == cand_only.timing.launches + 2
    assert [bytes(r) for r in both.candidate_corpus] == [bytes(r) for r in flagged.candidate_corpus]
    engine.score(C, 3, source=apo.SRC_ROLLOUTS, candidate_corpus=True)
    with pytest.raises(apo.ApoError):                                   # a failed call (K > C) leaves nothing readable
        engine.score(C, C + 1, source=apo.SRC_ROLLOUTS, candidate_corpus=True)
    with pytest.raises(apo.ApoError) as ei:
        engine.candidate_corpus_reports(0, C)
    assert ei.value.code == -3
    # every source without record fields: APO_E_ARG
    dims = orc.gen_dims(0x5EED0C23, 0, 2, 0, 4096, 300, 8)
    engine.dims_upload(dims)
    with pytest.raises(apo.ApoError) as ei:
        engine.score(2, 1, candidate_corpus=True)
    assert ei.value.code == -1
    engine.score_begin(2)
    with pytest.raises(apo.ApoError) as ei:
        engine.score_accumulate(0, candidate_corpus=True)
    assert ei.value.code == -1
    q8, d2, li, book = apo.compact_encode_host(dims)
    pc, pd, pbook, d2book = apo.packed_encode_host(dims)
    tl, th, tbook = apo.tuple_encode_host(pc, pd)
    flags = apo.engine.SCORE_CANDIDATE_CORPUS
    L, h = engine._L, engine._h
    o = apo.engine.ScoreOpts(1, apo.SRC_DIMS, flags, 0, 0, 0)
    s, n, k = np.empty(2), np.empty(2, np.uint64), np.empty(1, np.int32)
    p = apo.engine._p
    assert L.apo_score_host(h, o, p(dims), 2, 4096, p(s), p(n), p(k), None) == -1
    assert L.apo_score_host_compact(h, o, p(q8), p(d2), p(li), p(book), 2, 4096, p(s), p(n), p(k), None) == -1
    assert L.apo_score_host_packed(h, o, p(pc), p(pd), p(pbook), p(d2book), 2, 4096, p(s), p(n), p(k), None) == -1
    assert L.apo_score_host_tuples(h, o, p(tl), p(th), p(tbook[0]), p(tbook[1]), tbook[0].size, p(pbook), p(d2book), 2, 4096,
                                   p(s), p(n), p(k), None) == -1
    engine.tuples_upload(tl, th, tbook, pbook, d2book)
    with pytest.raises(apo.ApoError) as ei:
        engine.score(2, 1, source=apo.SRC_TUPLES, candidate_corpus=True)
    assert ei.value.code == -1
    engine.dims_upload_compact(dims)
    with pytest.raises(apo.ApoError) as ei:
        engine.score(2, 1, candidate_corpus=True)
    assert ei.value.code == -1


def test_generated_128x5M_r16_against_the_oracle(engine, orc, apo):
    seed, C, T = 0x5EED0C24, 128, 5_000_000
    engine.rollouts16_generate(seed, 0, C, 0, T, 300)
    res = engine.score(C, 4, source=apo.SRC_ROLLOUTS, candidate_corpus=True)
    for c in (0, 17, 38, 55, 73, 90, 111, 127):
        check_oracle(apo, res.candidate_corpus[c], orc.report(orc.gen_records(seed, orc.STREAM_ROLLOUT, c, 1, 0, T, 300, 16), nthreads=16))


def test_beam_search_hands_propose_the_pattern_report(engine, orc, apo):
    from importlib import import_module
    tcmod = import_module("senweaver-ide_b200.trace_collector")
    svcmod = import_module("senweaver-ide_b200.apo_service")
    svc = svcmod.APOService(engine, tcmod.TraceCollectorService(engine, storageService={}), storageService={})
    T = 2_000
    rows = {}

    def records(cands):
        out = np.stack([boundary_records(orc, 1, T, seed=1000 + int(c["version"][1:]))[0] for c in cands])
        for c, row in zip(cands, out):
            rows[c["version"]] = row
        return out

    seen = []

    def propose(parent, n, report=None):
        if report is not None:
            seen.append((parent["version"], report))
        return [parent["content"] + f"/{k}" for k in range(n)]

    svc.runBeamSearch("seed", propose, rolloutRecords=records, rounds=2, withReports=True)
    assert seen
    for version, report in seen:
        row = rows[version]
        ref = corpus_report_of(engine, apo, row)
        want = svc._emittedPatterns(ref, lambda p, gi: gi) + svc._dimensionPatterns(ref)
        strip = lambda ps: [{k: v for k, v in q.items() if k != "id"} for q in ps]
        assert strip(report["patterns"]) == strip(want), version
        assert report["byMode"] == svc._byMode(ref)
