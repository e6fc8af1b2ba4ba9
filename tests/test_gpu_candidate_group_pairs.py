"""Paired comparison per record group (APO_SCORE_CANDIDATE_GROUP_PAIRS, apo_candidate_group_pairs) on the H100, against
tests/group_pair_fixtures.py's exact model with no tolerance: every field by its bytes, NaN included.  Every call also sets
APO_SCORE_CANDIDATE_PAIRS and checks the invariants: summed over the labels every integer field is res.pairs' of the same
call, ref is the same in every group, and res.pairs itself satisfies pair_fixtures.invariants (mirrors, self-pairs, counts).
Every Form D route with and without recip, every source resident and streamed (the window boundary and R / R16 included),
windows off the 32-grid, sessions with reversed windows, candidate chunks and a window scored twice, custom and zero
weights, forced grids, many candidates at G = 64 and the flagship size; every combination of the seven per-candidate flags
with the flag-clear path unchanged; and the refusals."""
import importlib
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import group_pair_fixtures as gf
import pair_fixtures as pf
from extremes_fixtures import final_rewards
from test_gpu_candidate_pairs import ROUTES, eng, ref

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def check(got, model, where=""):
    """got [C][G] CandidatePair against the model [C][G] of dicts, every field by its bytes"""
    assert len(got) == len(model), where
    for c, (row, m) in enumerate(zip(got, model)):
        assert len(m) == len(row), where
        for g, x in enumerate(m):
            assert eng(row[g]) == ref(x), (where, c, g)


def check_call(engine, res, G, model=None, where=""):
    """the per-group pairs against the model and the invariants against the call's pairs"""
    if model is not None:
        check(res.group_pairs, model, where)
    counts = [int(x) for x in res.counts]
    pf.invariants(res.pairs, counts)
    gf.invariants(res.group_pairs, res.pairs, G)


def score(engine, C, K=1, **kw):
    return engine.score(C, K, pairs=True, group_pairs=True, **kw)


@pytest.mark.parametrize("recip", [False, True])
def test_fixtures_every_route(engine, orc, recip):
    """every fixture of group_pair_fixtures through K1, the Form W copy, the Form T copy (K1h whole rows by default, K1t and
    K1t2 forced); the extreme rows, outside the Form T domain, reach the routes that admit them"""
    try:
        for name, dims, refs, w, lab, G in gf.all_fixtures():
            engine.set_weights(orc.weights() if w is None else w)
            engine.candidate_refs_upload(refs)
            engine.record_groups_upload(lab, G)
            model = gf.model(dims, refs, lab, G, w, recip)
            for route, tune in ROUTES.items():
                if name.startswith("extreme") and route not in ("k1", "w_copy"):
                    continue
                engine.set_tuning(tune)
                engine.dims_upload(dims)
                check_call(engine, score(engine, dims.shape[0], recip=recip), G, model, (name, route))
    finally:
        engine.set_tuning(0)
        engine.set_weights(orc.weights())


def test_extreme_rows_past_2_128(engine, orc):
    """2^22 + 3 evaluations at 512 - 2^-15 against -512 under one label and under alternating labels: one (c, g) passes 2^83
    in D1 and 2^128 in D2; the mirror and two self-pairs"""
    import spread_fixtures as sf
    try:
        d = pf.extreme()
        T = d.shape[1]
        engine.set_weights(sf.w_one())
        for lab, G in ((np.zeros(T, np.uint8), 1), ((np.arange(T) % 2).astype(np.uint8), 2)):
            engine.record_groups_upload(lab, G)
            for refs in ([1, 0], [0, 1]):
                model = gf.model(d, refs, lab, G, sf.w_one())
                assert model[0][0]["D2"] > 2 ** 128 or refs == [0, 1]
                for route in ("k1", "w_copy"):
                    engine.set_tuning(ROUTES[route])
                    engine.dims_upload(d)
                    engine.candidate_refs_upload(refs)
                    check_call(engine, score(engine, 2), G, model, (G, refs, route))
    finally:
        engine.set_tuning(0)
        engine.set_weights(orc.weights())


def test_one_label_is_the_pairs_byte_for_byte(engine, orc, apo):
    C, T = 6, 50_001
    dims = orc.gen_dims(0x5EED7E01, 0, C, 0, T, 300, 8)
    dims[:, ::13] = np.nan
    dims[2, 7::19] = np.nan
    engine.candidate_refs_upload([pf.NONE, 0, 0, 3, 2, 5])
    engine.record_groups_upload(np.zeros(T, np.uint8), 1)
    for route, tune in ROUTES.items():
        engine.set_tuning(tune)
        engine.dims_upload(dims)
        res = score(engine, C)
        assert bytes(res.group_pairs) == bytes(res.pairs), route
    engine.set_tuning(0)


def test_every_source_and_the_streamed_calls(engine, orc, apo):
    C, T = 5, 70_003
    dims = orc.gen_dims(0x5EED7E02, 0, C, 0, T, 300, 8)
    dims[:, (np.arange(T) % 17) == 0] = np.nan
    dims[1, 5::23] = np.nan
    refs = np.array([pf.NONE, 0, 0, 4, 3], np.uint32)
    for kind in ("mod5", "lanes", "runs"):
        lab, G = gf.labels(kind, T)
        engine.candidate_refs_upload(refs)
        engine.record_groups_upload(lab, G)
        model = gf.model(dims, refs, lab, G)
        kw = dict(pairs=True, group_pairs=True)
        engine.dims_upload(dims)
        check_call(engine, engine.score(C, 2, **kw), G, model, kind)
        check_call(engine, engine.score_host(dims, 2, **kw), G, model, kind)                     # Form D streamed
        engine.dims_upload_compact(dims)
        check_call(engine, engine.score(C, 2, **kw), G, model, kind)                             # Form Q resident
        engine.dims_tuples()
        check_call(engine, engine.score(C, 2, source=apo.SRC_TUPLES, **kw), G, model, kind)      # device-built Form T
        q8, d2, li, book = apo.compact_encode_host(dims)
        check_call(engine, engine.score_host_compact(q8, d2, li, book, 2, **kw), G, model, kind)
        pc, pd, pbook, d2book = apo.packed_encode_host(dims)
        check_call(engine, engine.score_host_packed(pc, pd, pbook, d2book, 2, **kw), G, model, kind)
        tl, th, tbook = apo.tuple_encode_host(pc, pd)
        check_call(engine, engine.score_host_tuples(tl, th, tbook, pbook, d2book, 2, **kw), G, model, kind)
        engine.tuples_upload(tl, th, tbook, pbook, d2book)
        check_call(engine, engine.score(C, 2, source=apo.SRC_TUPLES, **kw), G, model, kind)      # uploaded Form T


def test_streamed_across_the_window_boundary(engine, orc, apo):
    """C = 256 rows of T = 180 001 through the host-streaming layouts: each row spans a 256 MB window boundary"""
    C, T = 256, 180_001
    dims = orc.gen_dims(0x5EED7E03, 0, C, 0, T, 300, 16)
    refs = np.array([pf.NONE if c % 5 == 0 else c - c % 5 for c in range(C)], np.uint32)
    lab, G = gf.labels("mod5", T)
    engine.candidate_refs_upload(refs)
    engine.record_groups_upload(lab, G)
    got = engine.score_host(dims, 2, pairs=True, group_pairs=True)
    check_call(engine, got, G)
    for c in (1, 128, 254):
        r = int(refs[c])
        m = gf.model(dims[[c, r]], [1, pf.NONE], lab, G)[0]
        check([got.group_pairs[c]], [[x | {"ref": r} for x in m]])
    q8, d2, li, book = apo.compact_encode_host(dims, nthreads=16)
    assert bytes(engine.score_host_compact(q8, d2, li, book, 2, pairs=True, group_pairs=True).group_pairs) == bytes(got.group_pairs)
    del q8, d2, li
    pc, pd, pbook, d2book = apo.packed_encode_host(dims, nthreads=16)
    del dims
    assert bytes(engine.score_host_packed(pc, pd, pbook, d2book, 2, pairs=True, group_pairs=True).group_pairs) == bytes(got.group_pairs)


def test_records_r_r16_resident_and_streamed(engine, orc, apo):
    C, T = 3, 9_001
    recs = orc.gen_records(0x5EED7E04, orc.STREAM_ROLLOUT, 0, C, 0, T, 300, 8)
    recs["flags"][:, ::7] &= ~np.uint8(8)
    recs["flags"][0, 3::11] &= ~np.uint8(8)
    refs = np.array([2, 0, 1], np.uint32)
    lab, G = gf.labels("ends", T)
    engine.candidate_refs_upload(refs)
    engine.record_groups_upload(lab, G)
    model = gf.rec_model(recs, refs, lab, G)
    engine.rollouts_upload(recs)
    check_call(engine, score(engine, C, 2, source=apo.SRC_ROLLOUTS), G, model)
    check_call(engine, engine.score_host_records(recs, 2, pairs=True, group_pairs=True), G, model)
    check_call(engine, score(engine, C, 2, source=apo.SRC_ROLLOUTS, recip=True), G, gf.rec_model(recs, refs, lab, G, recip=True))
    p16 = apo.pack16(recs)
    model16 = gf.rec_model(orc.unpack16(p16), refs, lab, G)
    engine.rollouts16_upload(p16)
    check_call(engine, score(engine, C, 2, source=apo.SRC_ROLLOUTS), G, model16)
    check_call(engine, engine.score_host_records(p16, 2, pairs=True, group_pairs=True), G, model16)
    C2, T2 = 64, 300_001                                  # across the window boundary (R: 131 072, R16: 262 144 records)
    big = orc.gen_records(0x5EED7E05, orc.STREAM_ROLLOUT, 0, C2, 0, T2, 300, 8)
    lab2, G2 = gf.labels("runs", T2)
    engine.record_groups_upload(lab2, G2)
    engine.candidate_refs_upload(np.array([C2 - 1] + [0] * (C2 - 1), np.uint32))
    got = engine.score_host_records(big, 2, pairs=True, group_pairs=True)
    check_call(engine, got, G2)
    m = gf.rec_model(big[[0, C2 - 1]], [1, 0], lab2, G2)
    check([got.group_pairs[0], got.group_pairs[C2 - 1]], [[x | {"ref": C2 - 1} for x in m[0]], [x | {"ref": 0} for x in m[1]]])
    assert bytes(engine.score_host_records(apo.pack16(big), 2, pairs=True, group_pairs=True).group_pairs) == bytes(got.group_pairs)


def test_windows_sessions_and_chunks(engine, orc, apo):
    C, T = 6, 40_000
    dims = orc.gen_dims(0x5EED7E06, 0, C, 0, T, 300, 8)
    dims[2, 100::9] = np.nan
    refs = np.array([1, 2, pf.NONE, 5, 3, 3], np.uint32)
    lab, G = gf.labels("mod5", T)
    engine.candidate_refs_upload(refs)
    engine.record_groups_upload(lab, G)
    engine.dims_upload(dims)
    fr, ok = final_rewards(dims)
    for first, count in ((4, 10_000), (36, 0), (1000, 33)):          # windows off the 32-grid: labels by absolute position
        end = T if count == 0 else first + count
        sel = np.zeros(T, bool)
        sel[first:end] = True
        check_call(engine, score(engine, C, first=first, count=count), G, gf.group_pair_model(fr, ok & sel, refs, lab, G), (first, count))
    whole = gf.model(dims, refs, lab, G)
    engine.score_begin(C)                                              # candidate chunks, windows in reverse order
    for c0 in (3, 0):
        engine.dims_upload(dims[c0:c0 + 3])
        engine.score_accumulate(c0, first=20_004, count=0, pairs=True, group_pairs=True)
        engine.score_accumulate(c0, first=0, count=20_004, pairs=True, group_pairs=True)
    res = engine.score_finish(C, 2, pairs=True, group_pairs=True)
    check_call(engine, res, G, whole)
    check(engine.score_finish(C, 2, pairs=True, group_pairs=True).group_pairs, whole)   # finish may be repeated
    engine.dims_upload(dims)                                           # the same window twice counts twice
    engine.score_begin(C)
    engine.score_accumulate(0, first=0, count=4096, group_pairs=True)
    engine.score_accumulate(0, first=0, count=4096, group_pairs=True)
    res = engine.score_finish(C, 1, group_pairs=True)
    twice = gf.group_pair_model(np.tile(fr[:, :4096], 2), np.tile(ok[:, :4096], 2), refs, np.tile(lab[:4096], 2), G)
    check(res.group_pairs, twice)
    assert res.pairs is None                                           # needs neither PAIRS nor GROUPS
    pc, pd, book, d2book = apo.packed_encode_host(dims)               # resident Form T windows
    tl, th, tbook = apo.tuple_encode_host(pc, pd)
    engine.tuples_upload(tl, th, tbook, book, d2book)
    engine.score_begin(C)
    engine.score_accumulate(0, source=apo.SRC_TUPLES, first=8200, count=0, group_pairs=True)
    engine.score_accumulate(0, source=apo.SRC_TUPLES, first=8, count=8192, group_pairs=True)
    sel = np.arange(T) >= 8
    check(engine.score_finish(C, 1, group_pairs=True).group_pairs, gf.group_pair_model(fr, ok & sel, refs, lab, G))


def test_refusals(engine, orc, apo):
    C, T = 4, 5000
    dims = orc.gen_dims(0x5EED7E07, 0, C, 0, T, 300, 8)
    engine.dims_upload(dims)
    lab, G = gf.labels("mod5", T)

    def code(fn, *a, **kw):
        with pytest.raises(apo.ApoError) as ei:
            fn(*a, **kw)
        return ei.value.code

    engine.candidate_refs_upload([1, 0, 3, 3])
    engine.record_groups_upload([])
    assert code(engine.score, C, 1, group_pairs=True) == -3            # no labels
    engine.record_groups_upload(lab[:4000], G)
    assert code(engine.score, C, 1, group_pairs=True) == -1            # a position past the labels' T
    engine.record_groups_upload(lab, G)
    engine.candidate_refs_upload([])
    assert code(engine.score, C, 1, group_pairs=True) == -3            # no refs
    engine.candidate_refs_upload([1, 0, 3, 3])
    engine.score(C, 1)
    assert code(engine.candidate_group_pairs, 0, C) == -3              # the last call did not set the flag
    res = engine.score(C, 1, group_pairs=True)
    check(res.group_pairs, gf.model(dims, [1, 0, 3, 3], lab, G))
    assert code(engine.candidate_group_pairs, 0, C, G + 1) == -1       # not the G it split by
    assert code(engine.candidate_group_pairs, C - 1, 2) == -1          # past its C
    assert len(engine.candidate_group_pairs(C, 0)) == 0
    assert code(engine.score, C, 1, first=2, group_pairs=True) == -1   # a failed call leaves nothing behind
    assert code(engine.candidate_group_pairs, 0, C) == -3
    engine.dims_upload(dims[:3])
    assert code(engine.score, 3, 1, group_pairs=True) == -1            # refs for C = 4, the call scores 3
    engine.dims_upload(dims)
    engine.score_begin(C)                                              # a mixed session
    engine.score_accumulate(0, first=0, count=2000, group_pairs=True)
    engine.score_accumulate(0, first=2000, count=0)
    assert code(engine.score_finish, C, 1, group_pairs=True) == -3
    for again in (lambda: engine.candidate_refs_upload([1, 0, 3, 3]), lambda: engine.record_groups_upload(lab, G)):
        engine.score_begin(C)                                          # refs or labels uploaded again mid-session
        engine.score_accumulate(0, first=0, count=2000, group_pairs=True)
        again()
        engine.score_accumulate(0, first=2000, count=0, group_pairs=True)
        assert code(engine.score_finish, C, 1, group_pairs=True) == -3
    engine.score_begin(C)                                              # a chunk whose candidate names a row outside it
    engine.candidate_refs_upload([1, 0, 0, 2])
    engine.dims_upload(dims[2:])
    assert code(engine.score_accumulate, 2, group_pairs=True) == -1
    engine.candidate_refs_upload([1, 0, 3, 2])
    engine.score_accumulate(2, group_pairs=True)
    engine.dims_upload(dims[:2])
    engine.score_accumulate(0, group_pairs=True)
    check(engine.score_finish(C, 1, group_pairs=True).group_pairs, gf.model(dims, [1, 0, 3, 2], lab, G))
    engine.dims_upload(dims)
    engine.score_begin(C + 1)                                          # C_total is not the refs' C
    assert code(engine.score_accumulate, 0, group_pairs=True) == -1
    check(engine.score(C, 1, count=64, group_pairs=True).group_pairs, gf.model(dims[:, :64], [1, 0, 3, 2], lab, G))


def test_flags_together_and_flag_clear_unchanged(engine, orc, apo):
    C, T, G = 5, 30_000, 6
    recs = orc.gen_records(0x5EED7E08, orc.STREAM_ROLLOUT, 0, C, 0, T, 300, 8)
    corpus = orc.gen_records(0x5EED7E08, orc.STREAM_CORPUS, 0, 1, 0, 3000, 300, 8).reshape(-1)
    labels = ((np.arange(T) // 37) % G).astype(np.uint8)
    refs = np.array([pf.NONE, 0, 0, 4, 3], np.uint32)
    engine.record_groups_upload(labels, G)
    engine.candidate_refs_upload(refs)
    engine.rollouts_upload(recs)
    engine.corpus_upload(corpus)
    model = gf.rec_model(recs, refs, labels, G)
    names = ("candidates", "candidate_corpus", "extremes", "groups", "spread", "pairs", "group_pairs")
    attrs = names[:6]

    def call(**kw):
        r = engine.score(C, 3, source=apo.SRC_ROLLOUTS, corpus=True, **kw)
        return r, (r.scores.tobytes(), r.counts.tobytes(), r.topk.tobytes(), bytes(r.report))

    plain, key = call()
    alone = {a: bytes(getattr(call(**{a: True})[0], a)) for a in attrs}
    for mask in range(128):
        flags = {f: bool(mask >> i & 1) for i, f in enumerate(names)}
        r, k = call(**flags)
        assert k == key, flags
        if flags["group_pairs"]:
            check(r.group_pairs, model)
        else:
            assert r.group_pairs is None
        for a in attrs:
            if flags[a]:
                assert bytes(getattr(r, a)) == alone[a], flags
    r, _ = call(group_pairs=True)
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
    for t in ({lanes!r}, {mod5!r}):
        e.record_groups_upload(np.load(t), int(np.load(t).max()) + 1)
        for tune in (0x10, 0x20, 0x40):
            e.set_tuning(tune)
            e.dims_upload(dims)
            out.append(bytes(e.score(dims.shape[0], 1, group_pairs=True).group_pairs).hex())
    e.close()
    sys.stdout.write(" ".join(out))
""")


def test_forced_grids(orc, tmp_path):
    """1 ... 7 CTAs (APO_K1_GRID, read once per process: a subprocess each): rows span several warps and flushes"""
    T = 3 * 1024 + 40
    d = orc.gen_dims(0x5EED7E09, 0, 4, 0, T, 300, 4)
    refs = [2, 2, 3, pf.NONE]
    path = str(tmp_path / "dims.npy")
    np.save(path, d)
    planes = {}
    for kind in ("lanes", "mod5"):
        planes[kind] = str(tmp_path / f"{kind}.npy")
        np.save(planes[kind], gf.labels(kind, T)[0])
    outs = None
    for g in range(1, 8):
        env = dict(os.environ, APO_K1_GRID=str(g))
        r = subprocess.run([sys.executable, "-c", GRID_SCRIPT.format(root=ROOT, path=path, refs=refs, lanes=planes["lanes"], mod5=planes["mod5"])],
                           env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr
        got = r.stdout.split()
        assert outs is None or got == outs, g
        outs = got
    CP = importlib.import_module("senweaver-ide_b200.engine").CandidatePair
    for i, kind in enumerate(("lanes", "mod5")):
        lab, G = gf.labels(kind, T)
        model = gf.model(d, refs, lab, G)
        for h in outs[3 * i:3 * i + 3]:
            check(((CP * G) * 4).from_buffer_copy(bytes.fromhex(h)), model, kind)


def test_custom_zero_and_recip_weights(engine, orc):
    C, T = 4, 20_000
    dims = orc.gen_dims(0x5EED7E0A, 0, C, 0, T, 300, 8)
    dims[:, ::5, 1:3] = np.nan
    refs = np.array([3, 0, 1, 2], np.uint32)
    lab, G = gf.labels("runs", T)
    engine.candidate_refs_upload(refs)
    engine.record_groups_upload(lab, G)
    try:
        for w in (np.array([0.0, 0.3, 0.0, 0.1, 0.2, 0.0, 0.1, 0.2, 0.1]), np.array([0.0] * 8 + [1.0]), np.linspace(0.05, 0.45, 9)):
            engine.set_weights(w)
            for tune in (0x10, 0):
                engine.set_tuning(tune)
                engine.dims_upload(dims)
                for recip in (False, True):
                    check_call(engine, score(engine, C, 2, recip=recip), G, gf.model(dims, refs, lab, G, w, recip), (tuple(w), tune, recip))
    finally:
        engine.set_tuning(0)
        engine.set_weights(orc.weights())


def test_many_candidates_at_64_groups(engine, orc):
    """C = 16384 at G = 64 (every lane its own label), every candidate naming candidate 0"""
    C, T = 16384, 200
    dims = orc.gen_dims(0x5EED7E0B, 0, C, 0, T, 300, 8)
    dims[:, ::3, :] = np.nan
    dims[1:5, :, :] = np.nan
    refs = np.zeros(C, np.uint32)
    lab, G = gf.labels("lanes", T)
    engine.candidate_refs_upload(refs)
    engine.record_groups_upload(lab, G)
    engine.dims_upload(dims)
    res = score(engine, C, 16)
    check_call(engine, res, G)
    sample = [0, 1, 5, 777, C - 1]
    fr, ok = final_rewards(dims[[0] + sample])
    m = gf.group_pair_model(fr, ok, [0] * (len(sample) + 1), lab, G)[1:]
    check([res.group_pairs[c] for c in sample], m)


def test_full_size_256x5M_against_the_generator(orc, apo):
    """config 3 (256 x 5 M resident Form D) through its default route and K1, byte-equal; sampled candidates against the model
    on the generator's rows.  On an engine of its own, closed at the end"""
    seed, C, T = 0x5EED0003, 256, 5_000_000
    refs = np.array([pf.NONE if c % 5 == 0 else c - c % 5 for c in range(C)], np.uint32)
    lab, G = gf.labels("mod5", T)
    engine = apo.Engine(0)
    try:
        engine.candidate_refs_upload(refs)
        engine.record_groups_upload(lab, G)
        engine.dims_generate(seed, 0, C, 0, T, 300)
        res = score(engine, C, 4)
        check_call(engine, res, G)
        engine.set_tuning(0x10)
        assert bytes(score(engine, C, 4).group_pairs) == bytes(res.group_pairs)
    finally:
        engine.close()
    for c in (1, 254):
        r = int(refs[c])
        rows = np.concatenate([orc.gen_dims(seed, c, 1, 0, T, 300, 16), orc.gen_dims(seed, r, 1, 0, T, 300, 16)])
        m = gf.model(rows, [1, pf.NONE], lab, G)[0]
        check([res.group_pairs[c]], [[x | {"ref": r} for x in m]])


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
            e.dims_generate(0x5EED7E0C, 0, C, rank * T, T, 300)
            e.candidate_refs_upload([1, 0, 3, 2])
            e.record_groups_upload(np.zeros(2 * T, np.uint8), 1)
            try:
                e.score(C, 1, group_pairs=True)
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
