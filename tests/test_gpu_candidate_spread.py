"""Per-candidate reward spread (APO_SCORE_CANDIDATE_SPREAD, apo_candidate_spread) on the H100, against
tests/spread_fixtures.py's exact model with no tolerance: every field by its bytes (NaN included), on every Form D route
with and without recip, every source, the host-streaming calls across their window boundary, windows off the 32-grid,
sessions with reversed windows, candidate chunks and a window scored twice, custom / zero weights, forced grids, many
candidates and the flagship size; n / S1 of every row against apo_debug_partials; every combination of the five
per-candidate flags with the flag-clear path unchanged; and the refusals.  The run-limit flush at one CTA is checked by
tests/test_gpu_cand_spread_flush.py."""
import importlib
import os
import struct
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import spread_fixtures as sf
from extremes_fixtures import final_rewards

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def bits(v) -> bytes:
    return struct.pack("<d", float(v))


def eng(s) -> tuple:
    return (int(s.n), int(s.sumLo), int(s.sumHi), int(s.sumSq[0]), int(s.sumSq[1]), int(s.sumSq[2]), bits(s.mean), bits(s.rewardSumSq),
            bits(s.variance), bits(s.stdDev), bits(s.stdErr))


def ref(m: dict) -> tuple:
    return tuple(bits(m[f]) if isinstance(m[f], float) else int(m[f]) for f in sf.FIELDS)


def check(got, model, where=""):
    assert len(got) == len(model), where
    for c, (s, m) in enumerate(zip(got, model)):
        assert eng(s) == ref(m), (where, c)


def check_call(engine, res, model=None, where=""):
    """the spreads against the model, and n / S1 / mean of every row against the call's own partials and scores"""
    if model is not None:
        check(res.spread, model, where)
    sums, counts = engine.debug_partials(len(res.spread))
    for c, s in enumerate(res.spread):
        assert (s.sum, int(s.n)) == (sums[c], counts[c]) == (sums[c], int(res.counts[c])), (where, c)
        assert s.n == 0 or bits(s.mean) == bits(res.scores[c]), (where, c)


ROUTES = {"k1": 0x10, "w_copy": 0x20, "t_copy": 0x40, "t_copy_k1t": 0x40 | 0x80 | 0x100, "t_copy_k1t2": 0x40 | 0x100}


@pytest.mark.parametrize("recip", [False, True])
def test_fixtures_every_route(engine, orc, apo, recip):
    """Form D through K1, the Form W copy and the Form T copy (whole rows through K1h by default, K1t and K1t2 forced); the
    const512 rows, outside the Form T domain, reach the routes that admit them"""
    try:
        for name, dims, w in sf.all_fixtures():
            engine.set_weights(orc.weights() if w is None else w)
            model = sf.model(dims, w, recip)
            for route, tune in ROUTES.items():
                engine.set_tuning(tune)
                engine.dims_upload(dims)
                res = engine.score(dims.shape[0], 1, recip=recip, spread=True)
                check_call(engine, res, model, (name, route))
    finally:
        engine.set_tuning(0)
        engine.set_weights(orc.weights())


def test_wide_rows_past_2_128(engine, orc):
    """one row of 2^22 + 3 evaluations at -(2 - 2^-23) (S2 past 2^128) on every route, and the one-unit row at 2^23 + 5
    evaluations, where M = n - 1 comes out of sums past 2^128"""
    try:
        d = sf.const2_wide()
        engine.set_weights(sf.w_one())
        m = [sf.constant_model(d.shape[1], -sf.F32_BELOW_2)]
        assert m[0]["S2"] > 2 ** 128
        for route, tune in ROUTES.items():
            engine.set_tuning(tune)
            engine.dims_upload(d)
            check_call(engine, engine.score(1, 1, spread=True), m, route)
        u = sf.one_unit((1 << 23) + 5, at=(1 << 22) + 17)
        engine.set_weights(sf.w_one_unit())
        mu = sf.model(u, sf.w_one_unit())
        assert mu[0]["M"] == mu[0]["n"] - 1 and mu[0]["S2"] > 2 ** 128
        for route, tune in (("k1", 0x10), ("default", 0)):
            engine.set_tuning(tune)
            engine.dims_upload(u)
            check_call(engine, engine.score(1, 1, spread=True), mu, route)
    finally:
        engine.set_tuning(0)
        engine.set_weights(orc.weights())


def test_every_source_and_the_streamed_calls(engine, orc, apo):
    C, T = 3, 70_003
    dims = orc.gen_dims(0x5EED7E01, 0, C, 0, T, 300, 8)
    dims[:, (np.arange(T) % 17) == 0] = np.nan
    model = sf.model(dims)
    engine.dims_upload(dims)
    check_call(engine, engine.score(C, 2, spread=True), model)
    check_call(engine, engine.score_host(dims, 2, spread=True), model)                          # Form D streamed
    engine.dims_upload_compact(dims)
    check_call(engine, engine.score(C, 2, spread=True), model)                                  # Form Q resident
    engine.dims_tuples()
    check_call(engine, engine.score(C, 2, source=apo.SRC_TUPLES, spread=True), model)           # device-built Form T
    q8, d2, li, book = apo.compact_encode_host(dims)
    check_call(engine, engine.score_host_compact(q8, d2, li, book, 2, spread=True), model)      # Form Q streamed
    pc, pd, pbook, d2book = apo.packed_encode_host(dims)
    check_call(engine, engine.score_host_packed(pc, pd, pbook, d2book, 2, spread=True), model)  # Form P streamed
    tl, th, tbook = apo.tuple_encode_host(pc, pd)
    check_call(engine, engine.score_host_tuples(tl, th, tbook, pbook, d2book, 2, spread=True), model)
    engine.tuples_upload(tl, th, tbook, pbook, d2book)
    check_call(engine, engine.score(C, 2, source=apo.SRC_TUPLES, spread=True), model)           # uploaded Form T


def test_streamed_across_the_window_boundary(engine, orc, apo):
    """C = 256 rows of T = 180 001 through every host-streaming layout: each row spans a 256 MB window boundary"""
    C, T = 256, 180_001
    dims = orc.gen_dims(0x5EED7E02, 0, C, 0, T, 300, 16)
    got = engine.score_host(dims, 2, spread=True)
    check_call(engine, got)
    for c in (0, 128, 255):
        check([got.spread[c]], sf.model(dims[c:c + 1]))
    q8, d2, li, book = apo.compact_encode_host(dims, nthreads=16)
    assert bytes(engine.score_host_compact(q8, d2, li, book, 2, spread=True).spread) == bytes(got.spread)
    del q8, d2, li
    pc, pd, pbook, d2book = apo.packed_encode_host(dims, nthreads=16)
    del dims
    assert bytes(engine.score_host_packed(pc, pd, pbook, d2book, 2, spread=True).spread) == bytes(got.spread)
    tl, th, tbook = apo.tuple_encode_host(pc, pd, nthreads=16)
    assert bytes(engine.score_host_tuples(tl, th, tbook, pbook, d2book, 2, spread=True).spread) == bytes(got.spread)


def test_records_r_r16_resident_and_streamed(engine, orc, apo):
    C, T = 3, 9_001
    recs = orc.gen_records(0x5EED7E03, orc.STREAM_ROLLOUT, 0, C, 0, T, 300, 8)
    recs["flags"][:, ::7] &= ~np.uint8(8)                 # without VALID: no reward
    model = sf.rec_model(recs)
    engine.rollouts_upload(recs)
    check_call(engine, engine.score(C, 2, source=apo.SRC_ROLLOUTS, spread=True), model)
    check_call(engine, engine.score_host_records(recs, 2, spread=True), model)
    check_call(engine, engine.score(C, 2, source=apo.SRC_ROLLOUTS, recip=True, spread=True), sf.rec_model(recs, recip=True))
    p16 = apo.pack16(recs)
    model16 = sf.rec_model(orc.unpack16(p16))
    engine.rollouts16_upload(p16)
    check_call(engine, engine.score(C, 2, source=apo.SRC_ROLLOUTS, spread=True), model16)
    check_call(engine, engine.score_host_records(p16, 2, spread=True), model16)
    C2, T2 = 64, 300_001                                  # across the window boundary (R: 131 072, R16: 262 144 records)
    big = orc.gen_records(0x5EED7E04, orc.STREAM_ROLLOUT, 0, C2, 0, T2, 300, 8)
    got = engine.score_host_records(big, 2, spread=True)
    check_call(engine, got)
    for c in (0, C2 - 1):
        check([got.spread[c]], sf.rec_model(big[c:c + 1]))
    assert bytes(engine.score_host_records(apo.pack16(big), 2, spread=True).spread) == bytes(got.spread)


def test_windows_sessions_and_chunks(engine, orc, apo):
    C, T = 6, 40_000
    dims = orc.gen_dims(0x5EED7E05, 0, C, 0, T, 300, 8)
    engine.dims_upload(dims)
    for first, count in ((4, 10_000), (36, 0), (1000, 33)):          # windows off the 32-grid
        end = T if count == 0 else first + count
        check_call(engine, engine.score(C, 1, first=first, count=count, spread=True), sf.model(dims[:, first:end]))
    whole = sf.model(dims)
    engine.score_begin(C)                                              # candidate chunks, windows in reverse order
    for c0 in (3, 0):
        engine.dims_upload(dims[c0:c0 + 3])
        engine.score_accumulate(c0, first=20_004, count=0, spread=True)
        engine.score_accumulate(c0, first=0, count=20_004, spread=True)
    check(engine.score_finish(C, 2, spread=True).spread, whole)
    check(engine.score_finish(C, 2, spread=True).spread, whole)        # finish may be repeated
    engine.dims_upload(dims)                                           # the same window twice counts twice
    engine.score_begin(C)
    engine.score_accumulate(0, first=0, count=4096, spread=True)
    engine.score_accumulate(0, first=0, count=4096, spread=True)
    fr, ok = final_rewards(dims[:, :4096])
    two = sf.spread_model(np.tile(fr, 2), np.tile(ok, 2))
    res = engine.score_finish(C, 1, spread=True)
    check(res.spread, two)
    check_call(engine, res)
    pc, pd, book, d2book = apo.packed_encode_host(dims)               # resident Form T windows
    tl, th, tbook = apo.tuple_encode_host(pc, pd)
    engine.tuples_upload(tl, th, tbook, book, d2book)
    engine.score_begin(C)
    engine.score_accumulate(0, source=apo.SRC_TUPLES, first=8200, count=0, spread=True)
    engine.score_accumulate(0, source=apo.SRC_TUPLES, first=8, count=8192, spread=True)
    check(engine.score_finish(C, 1, spread=True).spread, sf.model(dims[:, 8:]))


def test_refusals(engine, orc, apo):
    C, T = 4, 5000
    dims = orc.gen_dims(0x5EED7E06, 0, C, 0, T, 300, 8)
    engine.dims_upload(dims)

    def code(fn, *a, **kw):
        with pytest.raises(apo.ApoError) as ei:
            fn(*a, **kw)
        return ei.value.code

    engine.score(C, 1)
    assert code(engine.candidate_spread, 0, C) == -3                   # the last call did not set the flag
    res = engine.score(C, 1, spread=True)
    check(res.spread, sf.model(dims))
    assert code(engine.candidate_spread, C - 1, 2) == -1               # past its C
    assert code(engine.candidate_spread, 0, C + 1) == -1
    assert len(engine.candidate_spread(C, 0)) == 0
    assert code(engine.score, C, 1, first=2, spread=True) == -1        # a failed call leaves no spreads behind
    assert code(engine.candidate_spread, 0, C) == -3
    engine.score_begin(C)                                              # a mixed session
    engine.score_accumulate(0, first=0, count=2000, spread=True)
    engine.score_accumulate(0, first=2000, count=0)
    assert code(engine.score_finish, C, 1, spread=True) == -3
    assert code(engine.candidate_spread, 0, C) == -3
    res = engine.score(C, 1, count=64, spread=True)
    check(res.spread, sf.model(dims[:, :64]))


def test_flags_together_and_flag_clear_unchanged(engine, orc, apo):
    C, T, G = 5, 30_000, 6
    recs = orc.gen_records(0x5EED7E07, orc.STREAM_ROLLOUT, 0, C, 0, T, 300, 8)
    corpus = orc.gen_records(0x5EED7E07, orc.STREAM_CORPUS, 0, 1, 0, 3000, 300, 8).reshape(-1)
    labels = ((np.arange(T) // 37) % G).astype(np.uint8)
    engine.record_groups_upload(labels, G)
    engine.rollouts_upload(recs)
    engine.corpus_upload(corpus)
    model = sf.rec_model(recs)
    names = ("candidates", "candidate_corpus", "extremes", "groups", "spread")
    attrs = ("candidates", "candidate_corpus", "extremes", "groups")

    def call(**kw):
        r = engine.score(C, 3, source=apo.SRC_ROLLOUTS, corpus=True, **kw)
        return r, (r.scores.tobytes(), r.counts.tobytes(), r.topk.tobytes(), bytes(r.report))

    plain, key = call()
    alone = {a: bytes(getattr(call(**{a: True})[0], a)) for a in attrs}
    for mask in range(32):
        flags = {f: bool(mask >> i & 1) for i, f in enumerate(names)}
        r, k = call(**flags)
        assert k == key, flags
        if flags["spread"]:
            check(r.spread, model)
        else:
            assert r.spread is None
        for a in attrs:
            if flags[a]:
                assert bytes(getattr(r, a)) == alone[a], flags
    r, _ = call(spread=True)
    assert r.timing.launches == plain.timing.launches + 2                 # the pass and its report
    again, k2 = call()
    assert k2 == key and again.timing.launches == plain.timing.launches


GRID_SCRIPT = textwrap.dedent("""
    import sys, numpy as np
    sys.path.insert(0, {root!r})
    import importlib
    apo = importlib.import_module("senweaver-ide_b200")
    e = apo.Engine(0)
    dims = np.load({path!r})
    out = []
    for tune in (0x10, 0x20, 0x40):
        e.set_tuning(tune)
        e.dims_upload(dims)
        out.append(bytes(e.score(dims.shape[0], 1, spread=True).spread).hex())
    e.close()
    sys.stdout.write(" ".join(out))
""")


def test_forced_grids(orc, apo, tmp_path):
    """1 ... 7 CTAs (APO_K1_GRID, read once per process: a subprocess each): rows span several warps and flushes"""
    T = 3 * 1024 + 40
    d = orc.gen_dims(0x5EED7E08, 0, 3, 0, T, 300, 4)
    path = str(tmp_path / "dims.npy")
    np.save(path, d)
    outs = set()
    for g in range(1, 8):
        env = dict(os.environ, APO_K1_GRID=str(g))
        r = subprocess.run([sys.executable, "-c", GRID_SCRIPT.format(root=ROOT, path=path)], env=env, capture_output=True, text=True,
                           timeout=600)
        assert r.returncode == 0, r.stderr
        outs.update(r.stdout.split())
    assert len(outs) == 1
    got = (importlib.import_module("senweaver-ide_b200.engine").CandidateSpread * 3).from_buffer_copy(bytes.fromhex(outs.pop()))
    check(got, sf.model(d))


def test_custom_zero_and_recip_weights(engine, orc, apo):
    C, T = 4, 20_000
    dims = orc.gen_dims(0x5EED7E09, 0, C, 0, T, 300, 8)
    dims[:, ::5, 1:3] = np.nan
    try:
        for w in (np.array([0.0, 0.3, 0.0, 0.1, 0.2, 0.0, 0.1, 0.2, 0.1]), np.array([0.0] * 8 + [1.0]), np.linspace(0.05, 0.45, 9)):
            engine.set_weights(w)
            for tune in (0x10, 0):
                engine.set_tuning(tune)
                engine.dims_upload(dims)
                for recip in (False, True):
                    check_call(engine, engine.score(C, 2, recip=recip, spread=True), sf.model(dims, w, recip), (tuple(w), tune, recip))
    finally:
        engine.set_tuning(0)
        engine.set_weights(orc.weights())


def test_many_candidates(engine, orc):
    C, T = 16384, 96
    dims = orc.gen_dims(0x5EED7E0A, 0, C, 0, T, 300, 8)
    dims[:, ::3, :] = np.nan
    dims[:5, :, :] = np.nan                                            # n = 0
    dims[5, 1:, :] = np.nan                                            # n = 1
    engine.dims_upload(dims)
    res = engine.score(C, 16, spread=True)
    check_call(engine, res, sf.model(dims))


def test_full_size_256x5M_against_the_generator(orc, apo):
    """config 3 (256 x 5 M, 46 GB Form D resident) through its default route, byte-equal to K1; sampled rows against the model
    on the generator's rows, n / S1 of every row against the call's partials.  On an engine of its own, closed at the end: an
    engine's buffers only grow, and the session's shared engine would otherwise keep the 46 GB for every later test"""
    seed, C, T = 0x5EED0003, 256, 5_000_000
    engine = apo.Engine(0)
    try:
        engine.dims_generate(seed, 0, C, 0, T, 300)
        res = engine.score(C, 4, spread=True)
        check_call(engine, res)
        engine.set_tuning(0x10)
        res_k1 = engine.score(C, 4, spread=True)
        assert bytes(res_k1.spread) == bytes(res.spread)
    finally:
        engine.close()
    for c in (0, 85, 170, 255):
        check([res.spread[c]], sf.model(orc.gen_dims(seed, c, 1, 0, T, 300, 16)))


def test_multi_rank_refusal(orc, apo):
    """two handles joined into one communicator (one per GPU): a flagged call is refused with APO_E_STATE on every rank
    before anything is launched, and the flag-clear call still joins"""
    import threading
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    uid = apo.Engine.comm_unique_id()
    C, T, world, out, errs = 4, 4096, 2, {}, []

    def run(rank):
        try:
            e = apo.Engine(rank)
            e.comm_init(world, rank, uid)
            e.dims_generate(0x5EED7E0B, 0, C, rank * T, T, 300)
            try:
                e.score(C, 1, spread=True)
                out[rank] = "accepted"
            except apo.ApoError as ex:
                out[rank] = ex.code
            e.score(C, 1)
            e.close()
        except Exception as ex:
            errs.append((rank, repr(ex)))

    th = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=300)
    assert not errs, errs
    assert all(not t.is_alive() for t in th)
    assert out == {0: -3, 1: -3}
