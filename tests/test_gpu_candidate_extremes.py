"""Per-candidate extremes (APO_SCORE_CANDIDATE_EXTREMES, apo_candidate_extremes) on the H100, against the models of
tests/extremes_fixtures.py with no tolerance: positions, counts and every reward bit for bit, on every source and route,
the host-streaming calls across their window boundary, windows off the 32-grid, sessions with reversed windows and
candidate chunks, custom / zero / recip weights, forced grids, many candidates and the flagship size; and the flag-clear
path unchanged."""
import importlib
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import extremes_fixtures as xf

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def eng(x) -> dict:
    return {"n": int(x.n), "lowest": list(x.lowest), "highest": list(x.highest),
            "lowestReward": [np.float64(v).tobytes() for v in x.lowestReward],
            "highestReward": [np.float64(v).tobytes() for v in x.highestReward]}


def ref(m: dict) -> dict:
    return dict(m, lowestReward=[np.float64(v).tobytes() for v in m["lowestReward"]],
                highestReward=[np.float64(v).tobytes() for v in m["highestReward"]])


def check(res_ext, model):
    assert len(res_ext) == len(model)
    for c, (x, m) in enumerate(zip(res_ext, model)):
        assert eng(x) == ref(m), c


def rec_model(recs, w=None, recip=False, idx_base=0):
    fr, ok = xf.record_final_rewards(recs, w, recip)
    return [xf.extremes_sorted(fr[c], ok[c], idx_base + np.arange(fr.shape[1])) for c in range(fr.shape[0])]


ROUTES = {"k1": 0x10, "w_copy": 0x20, "t_copy": 0x40, "t_copy_k1t": 0x40 | 0x80 | 0x100, "t_copy_k1t2": 0x40 | 0x100}


@pytest.mark.parametrize("recip", [False, True])
def test_fixtures_every_route(engine, orc, apo, recip):
    """Form D through K1, the Form W copy and the Form T copy (forced beside it, with and without its counts and index plane)"""
    try:
        for name, dims, w in xf.all_fixtures():
            engine.set_weights(orc.weights() if w is None else w)
            model = xf.model(dims, w, recip)
            for route, tune in ROUTES.items():
                engine.set_tuning(tune)
                engine.dims_upload(dims)
                res = engine.score(dims.shape[0], 1, recip=recip, extremes=True)
                check(res.extremes, model)
                assert [x.n for x in res.extremes] == [min(32, int(n)) for n in res.counts], (name, route)
    finally:
        engine.set_tuning(0)
        engine.set_weights(orc.weights())


def test_every_source_and_the_streamed_calls(engine, orc, apo):
    C, T = 3, 70_003
    dims = orc.gen_dims(0x5EED0E01, 0, C, 0, T, 300, 8)
    dims[:, (np.arange(T) % 17) == 0] = np.nan
    model = xf.model(dims)
    engine.dims_upload(dims)
    check(engine.score(C, 2, extremes=True).extremes, model)
    check(engine.score_host(dims, 2, extremes=True).extremes, model)                          # Form D streamed
    engine.dims_upload_compact(dims)
    check(engine.score(C, 2, extremes=True).extremes, model)                                  # Form Q resident
    engine.dims_tuples()
    check(engine.score(C, 2, source=apo.SRC_TUPLES, extremes=True).extremes, model)           # device-built Form T
    q8, d2, li, book = apo.compact_encode_host(dims)
    check(engine.score_host_compact(q8, d2, li, book, 2, extremes=True).extremes, model)      # Form Q streamed
    pc, pd, pbook, d2book = apo.packed_encode_host(dims)
    check(engine.score_host_packed(pc, pd, pbook, d2book, 2, extremes=True).extremes, model)  # Form P streamed
    tl, th, tbook = apo.tuple_encode_host(pc, pd)
    check(engine.score_host_tuples(tl, th, tbook, pbook, d2book, 2, extremes=True).extremes, model)
    engine.tuples_upload(tl, th, tbook, pbook, d2book)
    check(engine.score(C, 2, source=apo.SRC_TUPLES, extremes=True).extremes, model)           # uploaded Form T


def test_streamed_across_the_window_boundary(engine, orc, apo):
    """C = 256 rows of T = 180 001: every host-streaming layout (D 36 B, Q 14 B, P 6 B, T 3 B per evaluation) needs more
    than one 256 MB window, so every row spans a window boundary; three rows against the model, all rows across layouts"""
    C, T = 256, 180_001
    dims = orc.gen_dims(0x5EED0E02, 0, C, 0, T, 300, 16)
    picks = (0, 128, 255)
    model = [xf.model(dims[c:c + 1])[0] for c in picks]
    got = engine.score_host(dims, 2, extremes=True).extremes
    assert [eng(got[c]) for c in picks] == [ref(m) for m in model]
    q8, d2, li, book = apo.compact_encode_host(dims, nthreads=16)
    assert bytes(engine.score_host_compact(q8, d2, li, book, 2, extremes=True).extremes) == bytes(got)
    del q8, d2, li
    pc, pd, pbook, d2book = apo.packed_encode_host(dims, nthreads=16)
    del dims
    assert bytes(engine.score_host_packed(pc, pd, pbook, d2book, 2, extremes=True).extremes) == bytes(got)
    tl, th, tbook = apo.tuple_encode_host(pc, pd, nthreads=16)
    assert bytes(engine.score_host_tuples(tl, th, tbook, pbook, d2book, 2, extremes=True).extremes) == bytes(got)


def test_records_r_r16_resident_and_streamed(engine, orc, apo):
    C, T = 3, 9_001
    recs = orc.gen_records(0x5EED0E03, orc.STREAM_ROLLOUT, 0, C, 0, T, 300, 8)
    recs["flags"][:, ::7] &= ~np.uint8(8)                 # records without VALID never appear
    model = rec_model(recs)
    engine.rollouts_upload(recs)
    check(engine.score(C, 2, source=apo.SRC_ROLLOUTS, extremes=True).extremes, model)
    check(engine.score_host_records(recs, 2, extremes=True).extremes, model)
    check(engine.score(C, 2, source=apo.SRC_ROLLOUTS, recip=True, extremes=True).extremes, rec_model(recs, recip=True))
    p16 = apo.pack16(recs)
    model16 = rec_model(orc.unpack16(p16))
    engine.rollouts16_upload(p16)
    check(engine.score(C, 2, source=apo.SRC_ROLLOUTS, extremes=True).extremes, model16)
    check(engine.score_host_records(p16, 2, extremes=True).extremes, model16)
    # streamed across the window boundary: 256 MB / (C * row) records per window (R: 131 072, R16: 262 144)
    C2, T2 = 64, 300_001
    big = orc.gen_records(0x5EED0E04, orc.STREAM_ROLLOUT, 0, C2, 0, T2, 300, 8)
    got = engine.score_host_records(big, 2, extremes=True).extremes
    for c in (0, C2 - 1):
        fr, ok = xf.record_final_rewards(big[c])
        assert eng(got[c]) == ref(xf.extremes_sorted(fr, ok, np.arange(T2))), c
    assert bytes(engine.score_host_records(apo.pack16(big), 2, extremes=True).extremes) == bytes(got)


def test_windows_sessions_and_chunks(engine, orc, apo):
    C, T = 6, 40_000
    dims = orc.gen_dims(0x5EED0E05, 0, C, 0, T, 300, 8)
    fr, ok = xf.final_rewards(dims)
    pos = np.arange(T)
    # windows off the 32-grid
    engine.dims_upload(dims)
    for first, count in ((4, 10_000), (36, 0), (1000, 33)):
        end = T if count == 0 else first + count
        res = engine.score(C, 1, first=first, count=count, extremes=True)
        check(res.extremes, [xf.extremes_sorted(fr[c, first:end], ok[c, first:end], pos[first:end]) for c in range(C)])
    # a session: candidate chunks, windows in reverse order
    whole = xf.model(dims)
    engine.score_begin(C)
    for c0 in (3, 0):
        engine.dims_upload(dims[c0:c0 + 3])
        engine.score_accumulate(c0, first=20_004, count=0, extremes=True)
        engine.score_accumulate(c0, first=0, count=20_004, extremes=True)
    check(engine.score_finish(C, 2, extremes=True).extremes, whole)
    check(engine.score_finish(C, 2, extremes=True).extremes, whole)                # finish may be repeated
    # the same window twice: its evaluations are listed twice
    engine.dims_upload(dims)
    engine.score_begin(C)
    engine.score_accumulate(0, first=0, count=4096, extremes=True)
    engine.score_accumulate(0, first=0, count=4096, extremes=True)
    got = engine.score_finish(C, 1, extremes=True).extremes
    two = [xf.extremes_sorted(np.tile(fr[c, :4096], 2), np.tile(ok[c, :4096], 2), np.tile(pos[:4096], 2)) for c in range(C)]
    check(got, two)
    # resident Form T windows
    pc, pd, book, d2book = apo.packed_encode_host(dims)
    tl, th, tbook = apo.tuple_encode_host(pc, pd)
    engine.tuples_upload(tl, th, tbook, book, d2book)
    engine.score_begin(C)
    engine.score_accumulate(0, source=apo.SRC_TUPLES, first=8200, count=0, extremes=True)
    engine.score_accumulate(0, source=apo.SRC_TUPLES, first=8, count=8192, extremes=True)
    check(engine.score_finish(C, 1, extremes=True).extremes,
          [xf.extremes_sorted(fr[c, 8:], ok[c, 8:], pos[8:]) for c in range(C)])


def test_refusals(engine, orc, apo):
    C, T = 4, 5000
    dims = orc.gen_dims(0x5EED0E06, 0, C, 0, T, 300, 8)
    engine.dims_upload(dims)
    engine.score(C, 1)
    with pytest.raises(apo.ApoError) as ei:                              # the last call did not set the flag
        engine.candidate_extremes(0, C)
    assert ei.value.code == -3
    engine.score(C, 1, extremes=True)
    with pytest.raises(apo.ApoError) as ei:
        engine.candidate_extremes(C - 1, 2)
    assert ei.value.code == -1
    assert len(engine.candidate_extremes(1, 3)) == 3
    engine.score_begin(C)
    engine.score_accumulate(0, first=0, count=2000, extremes=True)
    engine.score_accumulate(0, first=2000, count=0)
    with pytest.raises(apo.ApoError) as ei:                              # a mixed session
        engine.score_finish(C, 1, extremes=True)
    assert ei.value.code == -3
    with pytest.raises(apo.ApoError) as ei:                              # a failed call leaves no lists behind
        engine.candidate_extremes(0, C)
    assert ei.value.code == -3


def test_flags_together_and_flag_clear_unchanged(engine, orc, apo):
    C, T = 5, 30_000
    recs = orc.gen_records(0x5EED0E07, orc.STREAM_ROLLOUT, 0, C, 0, T, 300, 8)
    corpus = orc.gen_records(0x5EED0E07, orc.STREAM_CORPUS, 0, 1, 0, 3000, 300, 8).reshape(-1)
    engine.rollouts_upload(recs)
    engine.corpus_upload(corpus)

    def call(**kw):
        r = engine.score(C, 3, source=apo.SRC_ROLLOUTS, corpus=True, **kw)
        return r, (r.scores.tobytes(), r.counts.tobytes(), r.topk.tobytes(), bytes(r.report))

    plain, key = call()
    for flags in ({"extremes": True}, {"extremes": True, "candidates": True}, {"extremes": True, "candidate_corpus": True},
                  {"extremes": True, "candidates": True, "candidate_corpus": True}):
        r, k = call(**flags)
        assert k == key, flags
        check(r.extremes, rec_model(recs))
        if flags.get("candidates"):
            assert bytes(r.candidates) == bytes(call(candidates=True)[0].candidates)
        if flags.get("candidate_corpus"):
            assert bytes(r.candidate_corpus) == bytes(call(candidate_corpus=True)[0].candidate_corpus)
    r, k = call(extremes=True)
    assert r.timing.launches == plain.timing.launches + 2                 # the pass and its merge
    again, k2 = call()
    assert k2 == key and again.timing.launches == plain.timing.launches and again.extremes is None


GRID_SCRIPT = textwrap.dedent("""
    import sys, numpy as np
    sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
    import importlib, extremes_fixtures as xf
    apo = importlib.import_module("senweaver-ide_b200")
    e = apo.Engine(0)
    dims = np.load({path!r})
    e.set_tuning(0x10)
    e.dims_upload(dims)
    out = e.score(dims.shape[0], 1, extremes=True).extremes
    e.close()
    sys.stdout.write(bytes(out).hex())
""")


def test_forced_grids(orc, apo, tmp_path):
    """1 ... 7 CTAs (APO_K1_GRID, read once per process: a subprocess each): a row spans several warps, and a 32nd / 33rd
    tie sits on a segment boundary; the bytes equal the model's and every grid's"""
    T = 3 * 1024 + 40
    d = np.repeat(xf.rows(T, d1=np.float32(0.25))[None], 3, axis=0)
    d[0, 1000:1100, 1] = -0.5                             # 100 ties of the lowest reward across warp ranges
    d[1] = xf.falling(T)[0]
    d[2, ::97, 1] = 0.75
    path = str(tmp_path / "dims.npy")
    np.save(path, d)
    model = xf.model(d)
    outs = set()
    for g in range(1, 8):
        env = dict(os.environ, APO_K1_GRID=str(g))
        script = GRID_SCRIPT.format(root=ROOT, tests=os.path.join(ROOT, "tests"), path=path)
        r = subprocess.run([sys.executable, "-c", script], env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr
        outs.add(r.stdout)
    assert len(outs) == 1
    got = (importlib.import_module("senweaver-ide_b200.engine").CandidateExtremes * 3).from_buffer_copy(bytes.fromhex(outs.pop()))
    check(got, model)


def test_custom_zero_and_recip_weights(engine, orc, apo):
    C, T = 4, 20_000
    dims = orc.gen_dims(0x5EED0E08, 0, C, 0, T, 300, 8)
    dims[:, ::5, 1:3] = np.nan
    try:
        for w in (np.array([0.0, 0.3, 0.0, 0.1, 0.2, 0.0, 0.1, 0.2, 0.1]), np.array([0.0] * 8 + [1.0]), np.linspace(0.05, 0.45, 9)):
            engine.set_weights(w)
            for tune in (0x10, 0):
                engine.set_tuning(tune)
                engine.dims_upload(dims)
                for recip in (False, True):
                    check(engine.score(C, 2, recip=recip, extremes=True).extremes, xf.model(dims, w, recip))
    finally:
        engine.set_tuning(0)
        engine.set_weights(orc.weights())


def test_many_candidates(engine, orc):
    C, T = 16384, 96
    dims = orc.gen_dims(0x5EED0E09, 0, C, 0, T, 300, 8)
    dims[:, ::3, :] = np.nan
    engine.dims_upload(dims)
    check(engine.score(C, 16, extremes=True).extremes, xf.model(dims))


def test_full_size_256x5M_against_the_generator(engine, orc, apo):
    """config 3 (256 x 5 M, 46 GB Form D resident) through its default route: 8 spread rows against the generator's rows"""
    seed, C, T = 0x5EED0003, 256, 5_000_000
    engine.dims_generate(seed, 0, C, 0, T, 300)
    res = engine.score(C, 4, extremes=True)
    engine.set_tuning(0x10)
    try:
        res_k1 = engine.score(C, 4, extremes=True)
    finally:
        engine.set_tuning(0)
    assert bytes(res_k1.extremes) == bytes(res.extremes)
    for c in (0, 37, 74, 111, 148, 185, 222, 255):
        d = orc.gen_dims(seed, c, 1, 0, T, 300, 16)
        assert eng(res.extremes[c]) == ref(xf.model(d)[0]), c


def test_multi_rank_refusal(orc, apo):
    """two handles joined into one communicator (one per GPU, on two threads of this process): a flagged call is refused
    with APO_E_STATE on every rank before anything is launched, and the flag-clear call still joins"""
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
            e.dims_generate(0x5EED0E0A, 0, C, rank * T, T, 300)
            try:
                e.score(C, 1, extremes=True)
                out[rank] = "accepted"
            except apo.ApoError as ex:
                out[rank] = ex.code
            e.score(C, 1)
            e.close()
        except Exception as ex:                      # surfaced below: a failing thread must not hang the other silently
            errs.append((rank, repr(ex)))

    th = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=300)
    assert not errs, errs
    assert all(not t.is_alive() for t in th)
    assert out == {0: -3, 1: -3}
