"""Per-candidate breakdown (APO_SCORE_CANDIDATES, apo_candidate_reports) on the H100, against the CPU oracle
(oracle/candidates.py): integers, first-three examples and every binary64 field bit for bit, on every source, the
host-streaming calls, windowed / chunked sessions, custom and zero weights; and the flag-clear path unchanged."""
import math
import struct

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DIM_FIELDS = ("sum", "count", "avg", "low_flag", "low_severity", "sugg_flag", "sugg_priority")


@pytest.fixture(scope="module")
def oc(orc):
    from oracle import candidates
    candidates.build()
    return candidates


def _bits(x: float) -> bytes:
    return struct.pack("<d", x)


def eng_rep(r) -> dict:
    """engine CandidateReport -> the oracle's dict shape (floats as bit patterns)"""
    return {"total": r.total, "good": r.good, "bad": r.bad, "none": r.none, "goodRate": _bits(r.goodRate),
            "withReward": r.withReward, "rewardSum": _bits(r.rewardSum), "avgReward": _bits(r.avgReward),
            "dim": [{f: (_bits(getattr(r.dim[i], f)) if f in ("sum", "avg") else int(getattr(r.dim[i], f))) for f in DIM_FIELDS}
                    for i in range(9)],
            "badExamples": list(r.badExamples)}


def orc_rep(d: dict) -> dict:
    return {"total": d["total"], "good": d["good"], "bad": d["bad"], "none": d["none"], "goodRate": _bits(d["goodRate"]),
            "withReward": d["withReward"], "rewardSum": _bits(d["rewardSum"]), "avgReward": _bits(d["avgReward"]),
            "dim": [{f: (_bits(d["dim"][i][f]) if f in ("sum", "avg") else int(d["dim"][i][f])) for f in DIM_FIELDS} for i in range(9)],
            "badExamples": d["badExamples"]}


def assert_same(res_cands, ref, scores=None, counts=None):
    assert len(res_cands) == len(ref)
    for c, (r, d) in enumerate(zip(res_cands, ref)):
        assert eng_rep(r) == orc_rep(d), c
        if scores is not None:
            assert r.withReward == counts[c]
            if counts[c]:
                assert _bits(r.avgReward) == _bits(scores[c])           # avgReward == scores[c] bit for bit
            else:
                assert math.isnan(r.avgReward) and scores[c] == -math.inf


def eng_list(cands):
    return [eng_rep(r) for r in cands]


def dims_with_holes(orc, seed, C, T):
    """generator dims + NaN patterns: an all-null candidate, random absent dimensions, rows without d0"""
    rng = np.random.default_rng(seed)
    dims = orc.gen_dims(seed, 0, C, 0, T, 300, 8)
    holes = rng.random(dims.shape) < 0.05
    dims[holes] = np.nan
    dims[1] = np.nan                                              # a candidate without a single non-null evaluation
    return dims


def test_form_d_matches_oracle_and_scores(engine, orc, oc):
    C, T = 5, 10_001
    dims = dims_with_holes(orc, 0x5EED0C01, C, T)
    engine.dims_upload(dims)
    res = engine.score(C, 3, corpus=False, candidates=True)
    assert_same(res.candidates, oc.cand_dims(dims), res.scores, res.counts)
    assert res.candidates[1].withReward == 0 and list(res.candidates[1].badExamples) == [-1, -1, -1]
    assert math.isnan(res.candidates[1].avgReward)


def test_flag_clear_is_unchanged(engine, orc, apo):
    C, T = 6, 50_000
    dims = orc.gen_dims(0x5EED0C02, 0, C, 0, T, 300, 8)
    recs = orc.gen_records(0x5EED0C02, orc.STREAM_CORPUS, 0, 1, 0, 3000, 300, 8).reshape(-1)
    engine.dims_upload(dims)
    engine.corpus_upload(recs)

    def plain():
        r = engine.score(C, 3, corpus=True)
        return (r.scores.tobytes(), r.counts.tobytes(), r.topk.tobytes(), bytes(r.report), engine.debug_partials(C),
                r.timing.launches, r.candidates)

    before = plain()
    flagged = engine.score(C, 3, corpus=True, candidates=True)
    after = plain()
    assert before == after and before[-1] is None
    assert flagged.scores.tobytes() == before[0] and flagged.topk.tobytes() == before[2] and bytes(flagged.report) == before[3]
    assert flagged.timing.launches == before[5] + 2                     # the breakdown pass + its report kernel
    with pytest.raises(apo.ApoError) as ei:                             # the last scoring call did not set the flag
        engine.candidate_reports(0, C)
    assert ei.value.code == -3


def test_same_data_as_q_p_t_and_streamed_is_bit_identical(engine, orc, apo, oc):
    C, T = 4, 70_003
    dims = orc.gen_dims(0x5EED0C03, 0, C, 0, T, 300, 8)
    ref = [orc_rep(d) for d in oc.cand_dims(dims)]
    engine.dims_upload(dims)
    assert eng_list(engine.score(C, 2, candidates=True).candidates) == ref                        # Form D resident
    assert eng_list(engine.score_host(dims, 2, candidates=True).candidates) == ref                # Form D streamed
    engine.dims_upload_compact(dims)
    assert engine.dims_layout() == 2
    assert eng_list(engine.score(C, 2, candidates=True).candidates) == ref                        # Form Q resident
    q8, d2, li, book = apo.compact_encode_host(dims)
    assert eng_list(engine.score_host_compact(q8, d2, li, book, 2, candidates=True).candidates) == ref
    pc, pd, pbook, d2book = apo.packed_encode_host(dims)
    assert eng_list(engine.score_host_packed(pc, pd, pbook, d2book, 2, candidates=True).candidates) == ref   # Form P streamed
    tl, th, tbook = apo.tuple_encode_host(pc, pd)
    assert eng_list(engine.score_host_tuples(tl, th, tbook, pbook, d2book, 2, candidates=True).candidates) == ref
    engine.tuples_upload(tl, th, tbook, pbook, d2book)
    assert eng_list(engine.score(C, 2, source=apo.SRC_TUPLES, candidates=True).candidates) == ref     # Form T resident


def boundary_records(orc, C, T, seed=99):
    """the threshold-boundary records of the rollout parity test: every counter across its thresholds +-1"""
    rng = np.random.default_rng(seed)
    tokens = np.array([0, 1, 999, 1000, 1001, 1999, 2000, 2001, 4999, 5000, 5001, 9999, 10000, 10001, 14999, 15000, 15001, 29999, 30000, 30001,
                       31000, 31001, 65535, 10**6, 2**32 - 1], np.uint32)
    calls = np.array([0, 1, 2, 3, 4, 6, 7, 8, 9, 10, 11, 15, 16, 25, 26, 27, 62, 63, 64, 65, 100, 1000, 65535, 2**32 - 1], np.uint32)
    recs = np.zeros((C, T), orc.RECORD_DTYPE)
    recs["feedback"] = rng.integers(0, 4, (C, T))                                   # 3: not a feedback value -> none
    recs["flags"] = rng.integers(0, 4, (C, T)) | 8 | (rng.integers(0, 2, (C, T)) << 4)
    recs["flags"][rng.random((C, T)) < 0.03] &= ~np.uint8(8)
    recs["mode"] = rng.integers(0, 5, (C, T))
    recs["userMsgs"] = rng.integers(0, 12, (C, T))
    recs["asstMsgs"] = rng.integers(0, 12, (C, T))
    recs["toolCalls"] = calls[rng.integers(0, len(calls), (C, T))]
    fail = (rng.random((C, T)) * (np.minimum(recs["toolCalls"], 8) + 1)).astype(np.uint32)
    recs["toolFail"] = np.minimum(fail, recs["toolCalls"])
    recs["toolSucc"] = recs["toolCalls"] - recs["toolFail"]
    recs["llmCalls"] = rng.integers(0, 12, (C, T))
    recs["tokens"] = tokens[rng.integers(0, len(tokens), (C, T))]
    per = np.array([0, 1, 999.5, 1000, 1000.0001, 2999, 3000, 3001, 9999, 10000, 10001, 1e7], np.float64)
    recs["toolDurMs"] = (per[rng.integers(0, len(per), (C, T))] * np.maximum(recs["toolCalls"], 1)).astype(np.float32)
    return recs


def test_rollouts_r_r16_equal_oracle_and_the_corpus_report_of_each_row(engine, orc, apo, oc):
    C, T = 4, 24_000
    recs = boundary_records(orc, C, T)
    ref = oc.cand_records(recs)
    engine.rollouts_upload(recs)
    res = engine.score(C, 2, source=apo.SRC_ROLLOUTS, candidates=True)
    assert_same(res.candidates, ref, res.scores, res.counts)
    assert eng_list(engine.score_host_records(recs, 2, candidates=True).candidates) == [orc_rep(d) for d in ref]
    # a candidate row is a list of traces: its breakdown is the engine's corpus report of that row on every shared field
    for c in range(C):
        engine.corpus_upload(recs[c])
        rep = engine.score(C, 1, source=apo.SRC_ROLLOUTS, corpus=True).report
        b = res.candidates[c]
        for f in ("total", "good", "bad", "none", "withReward"):
            assert getattr(b, f) == getattr(rep, f), (c, f)
        for f in ("goodRate", "rewardSum", "avgReward"):
            assert _bits(getattr(b, f)) == _bits(getattr(rep, f)), (c, f)
        assert bytes(b.dim) == bytes(rep.dim), c
    # Form R16 (representable records: the generator's)
    gen = orc.gen_records(0x5EED0C04, orc.STREAM_ROLLOUT, 0, C, 0, 30_001, 300, 8)
    p16 = apo.pack16(gen)
    ref16 = [orc_rep(d) for d in oc.cand_records(orc.unpack16(p16))]
    engine.rollouts16_upload(p16)
    assert eng_list(engine.score(C, 2, source=apo.SRC_ROLLOUTS, candidates=True).candidates) == ref16
    assert eng_list(engine.score_host_records(p16, 2, candidates=True).candidates) == ref16


def test_windowed_sessions_and_candidate_chunks_equal_one_call(engine, orc, apo, oc):
    C, T = 6, 40_000
    dims = dims_with_holes(orc, 0x5EED0C05, C, T)
    ref = [orc_rep(d) for d in oc.cand_dims(dims)]
    engine.score_begin(C)
    for c0 in (0, 3):
        engine.dims_upload(dims[c0:c0 + 3])
        engine.score_accumulate(c0, first=0, count=16_000, candidates=True)
        engine.score_accumulate(c0, first=16_000, count=0, candidates=True)
    r1 = engine.score_finish(C, 2, candidates=True)
    assert eng_list(r1.candidates) == ref
    assert eng_list(engine.score_finish(C, 2, candidates=True).candidates) == ref     # finish may be repeated
    # windows arriving one by one: the breakdown so far is the breakdown of the records seen so far
    engine.dims_upload(dims)
    engine.score_begin(C)
    engine.score_accumulate(0, first=0, count=20_000, candidates=True)
    part = engine.score_finish(C, 2, candidates=True)
    assert eng_list(part.candidates) == [orc_rep(d) for d in oc.cand_dims(dims, T=20_000)]
    engine.score_accumulate(0, first=20_000, count=0, candidates=True)
    assert eng_list(engine.score_finish(C, 2, candidates=True).candidates) == ref
    # a mixed session refuses the breakdown; out-of-range requests are argument errors
    engine.score_begin(C)
    engine.score_accumulate(0, first=0, count=20_000, candidates=True)
    engine.score_accumulate(0, first=20_000, count=0)
    with pytest.raises(apo.ApoError) as ei:
        engine.score_finish(C, 2, candidates=True)
    assert ei.value.code == -3
    with pytest.raises(apo.ApoError) as ei:
        engine.candidate_reports(0, C)
    assert ei.value.code == -3
    engine.score(C, 2, candidates=True)
    with pytest.raises(apo.ApoError) as ei:
        engine.candidate_reports(C - 1, 2)
    assert ei.value.code == -1


def test_windowed_rollouts_and_tuples(engine, orc, apo, oc):
    C, T = 3, 33_000
    recs = boundary_records(orc, C, T, seed=7)
    engine.rollouts_upload(recs)
    engine.score_begin(C)
    engine.score_accumulate(0, source=apo.SRC_ROLLOUTS, first=12, count=10_000, candidates=True)
    r = engine.score_finish(C, 1, candidates=True)
    assert eng_list(r.candidates) == [orc_rep(d) for d in oc.cand_records(recs[:, 12:10_012], idx_base=12)]
    dims = orc.gen_dims(0x5EED0C06, 0, C, 0, T, 300, 8)
    pc, pd, book, d2book = apo.packed_encode_host(dims)
    tl, th, tbook = apo.tuple_encode_host(pc, pd)
    engine.tuples_upload(tl, th, tbook, book, d2book)
    engine.score_begin(C)
    engine.score_accumulate(0, source=apo.SRC_TUPLES, first=8, count=8192, candidates=True)
    engine.score_accumulate(0, source=apo.SRC_TUPLES, first=8200, count=0, candidates=True)
    r = engine.score_finish(C, 1, candidates=True)
    assert eng_list(r.candidates) == [orc_rep(d) for d in oc.cand_dims(dims[:, 8:], idx_base=8)]


def test_custom_and_zero_weights(engine, orc, oc):
    C, T = 4, 20_000
    dims = dims_with_holes(orc, 0x5EED0C07, C, T)
    recs = boundary_records(orc, C, 8_000, seed=3)
    try:
        for w in (np.array([0.0, 0.3, 0.0, 0.1, 0.2, 0.0, 0.1, 0.2, 0.1]), np.array([0.0] * 8 + [1.0]), np.linspace(0.05, 0.45, 9)):
            engine.set_weights(w)
            engine.dims_upload(dims)
            res = engine.score(C, 2, candidates=True)
            assert_same(res.candidates, oc.cand_dims(dims, w=w), res.scores, res.counts)
            engine.rollouts_upload(recs)
            res = engine.score(C, 2, source=1, candidates=True)
            assert_same(res.candidates, oc.cand_records(recs, w=w), res.scores, res.counts)
    finally:
        engine.set_weights(orc.weights())


def test_many_candidates(engine, orc, oc):
    C, T = 16384, 96
    dims = dims_with_holes(orc, 0x5EED0C08, C, T)
    engine.dims_upload(dims)
    res = engine.score(C, 16, candidates=True)
    assert_same(res.candidates, oc.cand_dims(dims), res.scores, res.counts)


def test_full_size_256x5M_against_the_generator(engine, orc, apo, oc):
    """config 3 (256 x 5 M, 46 GB Form D resident), its Form Q copy and its Form T copy: a few candidates over the full record
    axis against the oracle's generator path, and all 256 breakdowns equal across the three layouts"""
    seed, C, T = 0x5EED0003, 256, 5_000_000
    picks = [0, 97, 255]
    ref = [orc_rep(d) for d in oc.cand_generated(seed, picks, 0, T, 300, nthreads=16)]
    engine.dims_generate(seed, 0, C, 0, T, 300)
    res = engine.score(C, 4, candidates=True)
    assert [eng_rep(res.candidates[c]) for c in picks] == ref
    engine.dims_generate_compact(seed, 0, C, 0, T, 300)
    res_q = engine.score(C, 4, candidates=True)
    assert eng_list(res_q.candidates) == eng_list(res.candidates)
    # Form T of the same tensor: Form P planes exported from the resident Form Q copy, encoded on the host, made resident
    pc, pd = np.empty((C, T), np.uint32), np.empty((C, T), np.uint16)
    for c in range(C):
        engine.dims_packed_download(c, 0, T, out=(pc[c], pd[c]))
    book, d2book = engine.dims_codebook(), engine.dims_d2book()
    tl, th, tbook = apo.tuple_encode_host(pc, pd, nthreads=16)
    del pc, pd
    engine.tuples_upload(tl, th, tbook, book, d2book)
    del tl, th
    res_t = engine.score(C, 4, source=apo.SRC_TUPLES, candidates=True)
    assert [eng_rep(res_t.candidates[c]) for c in picks] == ref
    assert eng_list(res_t.candidates) == eng_list(res.candidates)
