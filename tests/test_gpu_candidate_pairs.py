"""Paired comparison with a reference (APO_SCORE_CANDIDATE_PAIRS, apo_candidate_pairs) on the H100, against
tests/pair_fixtures.py's exact model with no tolerance: every field by its bytes (NaN included), and on every call the
invariants of pair_fixtures.invariants (counts, mirrors, self-pairs, D1 against apo_debug_partials where neither row has a
null).  Every Form D route with and without recip, every source, the host-streaming calls across their window boundary,
windows off the 32-grid, sessions with reversed windows, candidate chunks and a window scored twice, custom and zero
weights, forced grids, many candidates and the flagship size; every combination of the six per-candidate flags with the
flag-clear path unchanged; and the refusals."""
import importlib
import os
import struct
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import pair_fixtures as pf
import spread_fixtures as sf
from extremes_fixtures import final_rewards

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROUTES = {"k1": 0x10, "w_copy": 0x20, "t_copy": 0x40, "t_copy_k1t": 0x40 | 0x80 | 0x100, "t_copy_k1t2": 0x40 | 0x100, "default": 0}


def bits(v) -> bytes:
    return struct.pack("<d", float(v))


def eng(p) -> tuple:
    return (int(p.ref), int(p.n), int(p.wins), int(p.losses), int(p.ties), int(p.candOnly), int(p.refOnly), int(p.sumLo), int(p.sumHi),
            int(p.sumSq[0]), int(p.sumSq[1]), int(p.sumSq[2]), bits(p.meanDiff), bits(p.variance), bits(p.stdDev), bits(p.stdErr))


def ref(m: dict) -> tuple:
    return tuple(bits(m[f]) if isinstance(m[f], float) else int(m[f]) for f in pf.FIELDS)


def check(got, model, where=""):
    assert len(got) == len(model), where
    for c, (p, m) in enumerate(zip(got, model)):
        assert eng(p) == ref(m), (where, c)


def check_call(engine, res, model=None, where="", ok=None):
    """the pairs against the model, and the invariants against the call's counts and partials (ok: [C][T] non-null mask of a
    whole-row call, for the D1 = S1_c - S1_r check on null-free rows)"""
    if model is not None:
        check(res.pairs, model, where)
    sums, _ = engine.debug_partials(len(res.pairs))
    free = None if ok is None else [bool(np.all(o)) for o in ok]
    pf.invariants(res.pairs, [int(x) for x in res.counts], sums, free)


@pytest.mark.parametrize("recip", [False, True])
def test_fixtures_every_route(engine, orc, recip):
    """Form D through K1, the Form W copy, the Form T copy (K1h whole rows by default, K1t and K1t2 forced); the extreme rows,
    outside the Form T domain, reach the routes that admit them"""
    try:
        for name, dims, refs, w in pf.all_fixtures():
            engine.set_weights(orc.weights() if w is None else w)
            engine.candidate_refs_upload(refs)
            fr, ok = final_rewards(dims, w, recip)
            model = pf.pair_model(fr, ok, refs)
            for route, tune in ROUTES.items():
                if name.startswith("extreme") and route not in ("k1", "w_copy"):
                    continue
                engine.set_tuning(tune)
                engine.dims_upload(dims)
                res = engine.score(dims.shape[0], 1, recip=recip, pairs=True)
                check_call(engine, res, model, (name, route), ok)
    finally:
        engine.set_tuning(0)
        engine.set_weights(orc.weights())


def test_extreme_rows_past_2_128(engine, orc):
    """2^22 + 3 evaluations at 512 - 2^-15 against -512: D1 past 2^83, D2 past 2^128; the mirror and two self-pairs"""
    try:
        d = pf.extreme()
        n = d.shape[1]
        engine.set_weights(sf.w_one())
        pair = [pf.constant_pair(n, sf.F32_BELOW_512, -512.0, 1), pf.constant_pair(n, -512.0, sf.F32_BELOW_512, 0)]
        selfs = [pf.constant_pair(n, sf.F32_BELOW_512, sf.F32_BELOW_512, 0), pf.constant_pair(n, -512.0, -512.0, 1)]
        for route in ("k1", "w_copy"):
            engine.set_tuning(ROUTES[route])
            engine.dims_upload(d)
            engine.candidate_refs_upload([1, 0])
            check_call(engine, engine.score(2, 1, pairs=True), pair, route)
            engine.candidate_refs_upload([0, 1])
            check_call(engine, engine.score(2, 1, pairs=True), selfs, route)
    finally:
        engine.set_tuning(0)
        engine.set_weights(orc.weights())


def test_every_source_and_the_streamed_calls(engine, orc, apo):
    C, T = 5, 70_003
    dims = orc.gen_dims(0x5EED7F01, 0, C, 0, T, 300, 8)
    dims[:, (np.arange(T) % 17) == 0] = np.nan
    dims[1, 5::23] = np.nan
    refs = np.array([pf.NONE, 0, 0, 4, 3], np.uint32)
    engine.candidate_refs_upload(refs)
    model = pf.model(dims, refs)
    engine.dims_upload(dims)
    check_call(engine, engine.score(C, 2, pairs=True), model)
    check_call(engine, engine.score_host(dims, 2, pairs=True), model)                          # Form D streamed
    engine.dims_upload_compact(dims)
    check_call(engine, engine.score(C, 2, pairs=True), model)                                  # Form Q resident
    engine.dims_tuples()
    check_call(engine, engine.score(C, 2, source=apo.SRC_TUPLES, pairs=True), model)           # device-built Form T
    q8, d2, li, book = apo.compact_encode_host(dims)
    check_call(engine, engine.score_host_compact(q8, d2, li, book, 2, pairs=True), model)      # Form Q streamed
    pc, pd, pbook, d2book = apo.packed_encode_host(dims)
    check_call(engine, engine.score_host_packed(pc, pd, pbook, d2book, 2, pairs=True), model)  # Form P streamed
    tl, th, tbook = apo.tuple_encode_host(pc, pd)
    check_call(engine, engine.score_host_tuples(tl, th, tbook, pbook, d2book, 2, pairs=True), model)
    engine.tuples_upload(tl, th, tbook, pbook, d2book)
    check_call(engine, engine.score(C, 2, source=apo.SRC_TUPLES, pairs=True), model)           # uploaded Form T


def test_streamed_across_the_window_boundary(engine, orc, apo):
    """C = 256 rows of T = 180 001 through every host-streaming layout: each row spans a 256 MB window boundary"""
    C, T = 256, 180_001
    dims = orc.gen_dims(0x5EED7F02, 0, C, 0, T, 300, 16)
    refs = np.array([pf.NONE if c % 5 == 0 else c - c % 5 for c in range(C)], np.uint32)
    engine.candidate_refs_upload(refs)
    got = engine.score_host(dims, 2, pairs=True)
    check_call(engine, got)
    for c in (1, 128, 254):
        r = int(refs[c])
        check([got.pairs[c]], [pf.model(dims[[c, r]], [1, pf.NONE])[0] | {"ref": r}])
    q8, d2, li, book = apo.compact_encode_host(dims, nthreads=16)
    assert bytes(engine.score_host_compact(q8, d2, li, book, 2, pairs=True).pairs) == bytes(got.pairs)
    del q8, d2, li
    pc, pd, pbook, d2book = apo.packed_encode_host(dims, nthreads=16)
    del dims
    assert bytes(engine.score_host_packed(pc, pd, pbook, d2book, 2, pairs=True).pairs) == bytes(got.pairs)
    tl, th, tbook = apo.tuple_encode_host(pc, pd, nthreads=16)
    assert bytes(engine.score_host_tuples(tl, th, tbook, pbook, d2book, 2, pairs=True).pairs) == bytes(got.pairs)


def test_records_r_r16_resident_and_streamed(engine, orc, apo):
    C, T = 3, 9_001
    recs = orc.gen_records(0x5EED7F03, orc.STREAM_ROLLOUT, 0, C, 0, T, 300, 8)
    recs["flags"][:, ::7] &= ~np.uint8(8)                 # without VALID: no reward
    recs["flags"][0, 3::11] &= ~np.uint8(8)
    refs = np.array([2, 0, 1], np.uint32)
    engine.candidate_refs_upload(refs)
    model = pf.rec_model(recs, refs)
    engine.rollouts_upload(recs)
    check_call(engine, engine.score(C, 2, source=apo.SRC_ROLLOUTS, pairs=True), model)
    check_call(engine, engine.score_host_records(recs, 2, pairs=True), model)
    check_call(engine, engine.score(C, 2, source=apo.SRC_ROLLOUTS, recip=True, pairs=True), pf.rec_model(recs, refs, recip=True))
    p16 = apo.pack16(recs)
    model16 = pf.rec_model(orc.unpack16(p16), refs)
    engine.rollouts16_upload(p16)
    check_call(engine, engine.score(C, 2, source=apo.SRC_ROLLOUTS, pairs=True), model16)
    check_call(engine, engine.score_host_records(p16, 2, pairs=True), model16)
    C2, T2 = 64, 300_001                                  # across the window boundary (R: 131 072, R16: 262 144 records)
    big = orc.gen_records(0x5EED7F04, orc.STREAM_ROLLOUT, 0, C2, 0, T2, 300, 8)
    engine.candidate_refs_upload(np.array([C2 - 1] + [0] * (C2 - 1), np.uint32))
    got = engine.score_host_records(big, 2, pairs=True)
    check_call(engine, got)
    m = pf.rec_model(big[[0, C2 - 1]], [1, 0])
    check([got.pairs[0], got.pairs[C2 - 1]], [m[0] | {"ref": C2 - 1}, m[1] | {"ref": 0}])
    assert bytes(engine.score_host_records(apo.pack16(big), 2, pairs=True).pairs) == bytes(got.pairs)


def test_windows_sessions_and_chunks(engine, orc, apo):
    C, T = 6, 40_000
    dims = orc.gen_dims(0x5EED7F05, 0, C, 0, T, 300, 8)
    dims[2, 100::9] = np.nan
    refs = np.array([1, 2, pf.NONE, 5, 3, 3], np.uint32)   # every reference inside its chunk [0, 3) / [3, 6)
    engine.candidate_refs_upload(refs)
    engine.dims_upload(dims)
    for first, count in ((4, 10_000), (36, 0), (1000, 33)):          # windows off the 32-grid
        end = T if count == 0 else first + count
        check_call(engine, engine.score(C, 1, first=first, count=count, pairs=True), pf.model(dims[:, first:end], refs))
    whole = pf.model(dims, refs)
    engine.score_begin(C)                                              # candidate chunks, windows in reverse order
    for c0 in (3, 0):
        engine.dims_upload(dims[c0:c0 + 3])
        engine.score_accumulate(c0, first=20_004, count=0, pairs=True)
        engine.score_accumulate(c0, first=0, count=20_004, pairs=True)
    res = engine.score_finish(C, 2, pairs=True)
    check(res.pairs, whole)
    check_call(engine, res)
    check(engine.score_finish(C, 2, pairs=True).pairs, whole)         # finish may be repeated
    engine.dims_upload(dims)                                           # the same window twice counts twice
    engine.score_begin(C)
    engine.score_accumulate(0, first=0, count=4096, pairs=True)
    engine.score_accumulate(0, first=0, count=4096, pairs=True)
    fr, ok = final_rewards(dims[:, :4096])
    res = engine.score_finish(C, 1, pairs=True)
    check(res.pairs, pf.pair_model(np.tile(fr, 2), np.tile(ok, 2), refs))
    check_call(engine, res)
    pc, pd, book, d2book = apo.packed_encode_host(dims)               # resident Form T windows
    tl, th, tbook = apo.tuple_encode_host(pc, pd)
    engine.tuples_upload(tl, th, tbook, book, d2book)
    engine.score_begin(C)
    engine.score_accumulate(0, source=apo.SRC_TUPLES, first=8200, count=0, pairs=True)
    engine.score_accumulate(0, source=apo.SRC_TUPLES, first=8, count=8192, pairs=True)
    check(engine.score_finish(C, 1, pairs=True).pairs, pf.model(dims[:, 8:], refs))


def test_refusals(engine, orc, apo):
    C, T = 4, 5000
    dims = orc.gen_dims(0x5EED7F06, 0, C, 0, T, 300, 8)
    engine.dims_upload(dims)

    def code(fn, *a, **kw):
        with pytest.raises(apo.ApoError) as ei:
            fn(*a, **kw)
        return ei.value.code

    engine.candidate_refs_upload([])
    assert code(engine.score, C, 1, pairs=True) == -3                  # no refs
    assert code(engine.candidate_refs_upload, [1, 4, 0, 0]) == -1      # an entry >= C
    assert code(engine.score, C, 1, pairs=True) == -3                  # ... keeps the previous (none)
    engine.candidate_refs_upload([1, 0, 3, 3])
    assert code(engine.candidate_refs_upload, [1, 0, 9, pf.NONE]) == -1
    engine.score(C, 1)
    assert code(engine.candidate_pairs, 0, C) == -3                    # the last call did not set the flag
    res = engine.score(C, 1, pairs=True)                               # the refused upload kept [1, 0, 3, 3]
    check(res.pairs, pf.model(dims, [1, 0, 3, 3]))
    assert code(engine.candidate_pairs, C - 1, 2) == -1                # past its C
    assert len(engine.candidate_pairs(C, 0)) == 0
    assert code(engine.score, C, 1, first=2, pairs=True) == -1         # a failed call leaves no pairs behind
    assert code(engine.candidate_pairs, 0, C) == -3
    engine.dims_upload(dims[:3])
    assert code(engine.score, 3, 1, pairs=True) == -1                  # refs for C = 4, the call scores 3
    engine.dims_upload(dims)
    engine.score_begin(C)                                              # a mixed session
    engine.score_accumulate(0, first=0, count=2000, pairs=True)
    engine.score_accumulate(0, first=2000, count=0)
    assert code(engine.score_finish, C, 1, pairs=True) == -3
    assert code(engine.candidate_pairs, 0, C) == -3
    engine.score_begin(C)                                              # refs uploaded again mid-session
    engine.score_accumulate(0, first=0, count=2000, pairs=True)
    engine.candidate_refs_upload([1, 0, 3, 3])
    engine.score_accumulate(0, first=2000, count=0, pairs=True)
    assert code(engine.score_finish, C, 1, pairs=True) == -3
    engine.score_begin(C)                                              # a chunk whose candidate names a row outside it
    engine.candidate_refs_upload([1, 0, 0, 2])
    engine.dims_upload(dims[2:])
    assert code(engine.score_accumulate, 2, pairs=True) == -1
    engine.candidate_refs_upload([1, 0, 3, 2])
    engine.score_accumulate(2, pairs=True)
    engine.dims_upload(dims[:2])
    engine.score_accumulate(0, pairs=True)
    check(engine.score_finish(C, 1, pairs=True).pairs, pf.model(dims, [1, 0, 3, 2]))
    engine.dims_upload(dims)
    engine.score_begin(C + 1)                                          # C_total is not the refs' C
    assert code(engine.score_accumulate, 0, pairs=True) == -1
    res = engine.score(C, 1, count=64, pairs=True)
    check(res.pairs, pf.model(dims[:, :64], [1, 0, 3, 2]))


def test_flags_together_and_flag_clear_unchanged(engine, orc, apo):
    C, T, G = 5, 30_000, 6
    recs = orc.gen_records(0x5EED7F07, orc.STREAM_ROLLOUT, 0, C, 0, T, 300, 8)
    corpus = orc.gen_records(0x5EED7F07, orc.STREAM_CORPUS, 0, 1, 0, 3000, 300, 8).reshape(-1)
    labels = ((np.arange(T) // 37) % G).astype(np.uint8)
    refs = np.array([pf.NONE, 0, 0, 4, 3], np.uint32)
    engine.record_groups_upload(labels, G)
    engine.candidate_refs_upload(refs)
    engine.rollouts_upload(recs)
    engine.corpus_upload(corpus)
    model = pf.rec_model(recs, refs)
    names = ("candidates", "candidate_corpus", "extremes", "groups", "spread", "pairs")
    attrs = ("candidates", "candidate_corpus", "extremes", "groups", "spread")

    def call(**kw):
        r = engine.score(C, 3, source=apo.SRC_ROLLOUTS, corpus=True, **kw)
        return r, (r.scores.tobytes(), r.counts.tobytes(), r.topk.tobytes(), bytes(r.report))

    plain, key = call()
    alone = {a: bytes(getattr(call(**{a: True})[0], a)) for a in attrs}
    for mask in range(64):
        flags = {f: bool(mask >> i & 1) for i, f in enumerate(names)}
        r, k = call(**flags)
        assert k == key, flags
        if flags["pairs"]:
            check(r.pairs, model)
        else:
            assert r.pairs is None
        for a in attrs:
            if flags[a]:
                assert bytes(getattr(r, a)) == alone[a], flags
    r, _ = call(pairs=True)
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
    e.candidate_refs_upload(np.array({refs!r}, np.uint32))
    out = []
    for tune in (0x10, 0x20, 0x40):
        e.set_tuning(tune)
        e.dims_upload(dims)
        out.append(bytes(e.score(dims.shape[0], 1, pairs=True).pairs).hex())
    e.close()
    sys.stdout.write(" ".join(out))
""")


def test_forced_grids(orc, tmp_path):
    """1 ... 7 CTAs (APO_K1_GRID, read once per process: a subprocess each): rows span several warps and flushes"""
    T = 3 * 1024 + 40
    d = orc.gen_dims(0x5EED7F08, 0, 4, 0, T, 300, 4)
    refs = [2, 2, 3, pf.NONE]
    path = str(tmp_path / "dims.npy")
    np.save(path, d)
    outs = set()
    for g in range(1, 8):
        env = dict(os.environ, APO_K1_GRID=str(g))
        r = subprocess.run([sys.executable, "-c", GRID_SCRIPT.format(root=ROOT, path=path, refs=refs)], env=env, capture_output=True,
                           text=True, timeout=600)
        assert r.returncode == 0, r.stderr
        outs.update(r.stdout.split())
    assert len(outs) == 1
    got = (importlib.import_module("senweaver-ide_b200.engine").CandidatePair * 4).from_buffer_copy(bytes.fromhex(outs.pop()))
    check(got, pf.model(d, refs))


def test_custom_zero_and_recip_weights(engine, orc):
    C, T = 4, 20_000
    dims = orc.gen_dims(0x5EED7F09, 0, C, 0, T, 300, 8)
    dims[:, ::5, 1:3] = np.nan
    refs = np.array([3, 0, 1, 2], np.uint32)
    engine.candidate_refs_upload(refs)
    try:
        for w in (np.array([0.0, 0.3, 0.0, 0.1, 0.2, 0.0, 0.1, 0.2, 0.1]), np.array([0.0] * 8 + [1.0]), np.linspace(0.05, 0.45, 9)):
            engine.set_weights(w)
            for tune in (0x10, 0):
                engine.set_tuning(tune)
                engine.dims_upload(dims)
                for recip in (False, True):
                    check_call(engine, engine.score(C, 2, recip=recip, pairs=True), pf.model(dims, refs, w, recip), (tuple(w), tune, recip))
    finally:
        engine.set_tuning(0)
        engine.set_weights(orc.weights())


def test_many_candidates(engine, orc):
    """C = 16384, every candidate naming candidate 0"""
    C, T = 16384, 96
    dims = orc.gen_dims(0x5EED7F0A, 0, C, 0, T, 300, 8)
    dims[:, ::3, :] = np.nan
    dims[1:5, :, :] = np.nan                                           # n = 0
    dims[5, 1:, :] = np.nan                                            # n <= 1
    refs = np.zeros(C, np.uint32)
    engine.candidate_refs_upload(refs)
    engine.dims_upload(dims)
    res = engine.score(C, 16, pairs=True)
    check_call(engine, res, pf.model(dims, refs))


def test_full_size_256x5M_against_the_generator(orc, apo):
    """config 3 (256 x 5 M, 46 GB Form D resident) through its default route, byte-equal to K1; sampled pairs against the model
    on the generator's rows.  On an engine of its own, closed at the end"""
    seed, C, T = 0x5EED0003, 256, 5_000_000
    refs = np.array([pf.NONE if c % 5 == 0 else c - c % 5 for c in range(C)], np.uint32)
    engine = apo.Engine(0)
    try:
        engine.candidate_refs_upload(refs)
        engine.dims_generate(seed, 0, C, 0, T, 300)
        res = engine.score(C, 4, pairs=True)
        check_call(engine, res)
        engine.set_tuning(0x10)
        res_k1 = engine.score(C, 4, pairs=True)
        assert bytes(res_k1.pairs) == bytes(res.pairs)
    finally:
        engine.close()
    for c in (1, 254):
        r = int(refs[c])
        rows = np.concatenate([orc.gen_dims(seed, c, 1, 0, T, 300, 16), orc.gen_dims(seed, r, 1, 0, T, 300, 16)])
        check([res.pairs[c]], [pf.model(rows, [1, pf.NONE])[0] | {"ref": r}])


def test_multi_rank_refusal(orc, apo):
    """two handles joined into one communicator (one per GPU): a flagged call is refused with APO_E_STATE on every rank"""
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
            e.dims_generate(0x5EED7F0B, 0, C, rank * T, T, 300)
            e.candidate_refs_upload([1, 0, 3, 2])
            try:
                e.score(C, 1, pairs=True)
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
