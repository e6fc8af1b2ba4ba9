"""Per-candidate group scores (APO_SCORE_CANDIDATE_GROUPS, apo_record_groups_upload / apo_candidate_groups) on the H100,
against tests/group_fixtures.group_model with no tolerance: every field bit for bit, on every source and route, the
host-streaming calls across their window boundary, windows off the 32-grid, sessions with reversed windows, candidate
chunks and a window scored twice, custom / zero / recip weights, forced grids, many candidates with G = 64 and the
flagship size; G = 1 against the breakdown; every flag combination with the flag-clear path unchanged; and the refusals."""
import importlib
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import group_fixtures as gf
from extremes_fixtures import final_rewards

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ("total", "good", "bad", "goodRate", "withReward", "rewardSum", "avgReward")


def bits(v) -> bytes:
    return np.float64(v).tobytes()


def eng(s) -> tuple:
    return tuple(bits(getattr(s, f)) if isinstance(getattr(s, f), float) else int(getattr(s, f)) for f in FIELDS)


def ref(s: dict) -> tuple:
    return tuple(bits(s[f]) if isinstance(s[f], float) else int(s[f]) for f in FIELDS)


def check(got, model):
    assert len(got) == len(model)
    for c, (row, m) in enumerate(zip(got, model)):
        assert [eng(s) for s in row] == [ref(s) for s in m], c


def window_model(dims, labels, G, first, end, w=None, recip=False):
    fr, ok = final_rewards(dims[:, first:end], w, recip)
    return gf.group_model(fr, ok, gf.dims_tally(dims[:, first:end]), labels[first:end], G)


ROUTES = {"k1": 0x10, "w_copy": 0x20, "t_copy": 0x40, "t_copy_k1t": 0x40 | 0x80 | 0x100, "t_copy_k1t2": 0x40 | 0x100}


@pytest.mark.parametrize("recip", [False, True])
def test_fixtures_every_route(engine, orc, apo, recip):
    """Form D through K1, the Form W copy and the Form T copy (whole rows through K1h by default, K1t and K1t2 forced)"""
    try:
        for name, dims, labels, G, w in gf.all_fixtures() + [("wide",) + gf.wide() + (gf.w_d0(),)]:
            engine.set_weights(orc.weights() if w is None else w)
            engine.record_groups_upload(labels, G)
            model = gf.model(dims, labels, G, w, recip)
            for route, tune in ROUTES.items():
                engine.set_tuning(tune)
                engine.dims_upload(dims)
                res = engine.score(dims.shape[0], 1, recip=recip, groups=True, candidates=G == 1)
                check(res.groups, model)
                assert [sum(s.withReward for s in row) for row in res.groups] == [int(n) for n in res.counts], (name, route)
                if G == 1:                                                # every field of the breakdown, and scores[c]
                    for c, (row, r) in enumerate(zip(res.groups, res.candidates)):
                        s = row[0]
                        assert (s.total, s.good, s.bad, s.withReward) == (r.total, r.good, r.bad, r.withReward), (name, route, c)
                        assert bits(s.goodRate) == bits(r.goodRate) and bits(s.rewardSum) == bits(r.rewardSum)
                        assert bits(s.avgReward) == bits(r.avgReward) == bits(res.scores[c]) or r.withReward == 0
    finally:
        engine.set_tuning(0)
        engine.set_weights(orc.weights())


def test_every_source_and_the_streamed_calls(engine, orc, apo):
    C, T, G = 3, 70_003, 5
    dims = orc.gen_dims(0x5EED6E01, 0, C, 0, T, 300, 8)
    dims[:, (np.arange(T) % 17) == 0] = np.nan
    labels = ((np.arange(T) // 300) % G).astype(np.uint8)
    engine.record_groups_upload(labels, G)
    model = gf.model(dims, labels, G)
    engine.dims_upload(dims)
    check(engine.score(C, 2, groups=True).groups, model)
    check(engine.score_host(dims, 2, groups=True).groups, model)                          # Form D streamed
    engine.dims_upload_compact(dims)
    check(engine.score(C, 2, groups=True).groups, model)                                  # Form Q resident
    engine.dims_tuples()
    check(engine.score(C, 2, source=apo.SRC_TUPLES, groups=True).groups, model)           # device-built Form T
    q8, d2, li, book = apo.compact_encode_host(dims)
    check(engine.score_host_compact(q8, d2, li, book, 2, groups=True).groups, model)      # Form Q streamed
    pc, pd, pbook, d2book = apo.packed_encode_host(dims)
    check(engine.score_host_packed(pc, pd, pbook, d2book, 2, groups=True).groups, model)  # Form P streamed
    tl, th, tbook = apo.tuple_encode_host(pc, pd)
    check(engine.score_host_tuples(tl, th, tbook, pbook, d2book, 2, groups=True).groups, model)
    engine.tuples_upload(tl, th, tbook, pbook, d2book)
    check(engine.score(C, 2, source=apo.SRC_TUPLES, groups=True).groups, model)           # uploaded Form T


def test_streamed_across_the_window_boundary(engine, orc, apo):
    """C = 256 rows of T = 180 001 through every host-streaming layout: each row spans a 256 MB window boundary"""
    C, T, G = 256, 180_001, 64
    dims = orc.gen_dims(0x5EED6E02, 0, C, 0, T, 300, 16)
    labels = (np.arange(T) % G).astype(np.uint8)
    engine.record_groups_upload(labels, G)
    picks = (0, 128, 255)
    got = engine.score_host(dims, 2, groups=True).groups
    for c in picks:
        check([got[c]], gf.model(dims[c:c + 1], labels, G))
    q8, d2, li, book = apo.compact_encode_host(dims, nthreads=16)
    assert bytes(engine.score_host_compact(q8, d2, li, book, 2, groups=True).groups) == bytes(got)
    del q8, d2, li
    pc, pd, pbook, d2book = apo.packed_encode_host(dims, nthreads=16)
    del dims
    assert bytes(engine.score_host_packed(pc, pd, pbook, d2book, 2, groups=True).groups) == bytes(got)
    tl, th, tbook = apo.tuple_encode_host(pc, pd, nthreads=16)
    assert bytes(engine.score_host_tuples(tl, th, tbook, pbook, d2book, 2, groups=True).groups) == bytes(got)


def test_records_r_r16_resident_and_streamed(engine, orc, apo):
    C, T, G = 3, 9_001, 7
    recs = orc.gen_records(0x5EED6E03, orc.STREAM_ROLLOUT, 0, C, 0, T, 300, 8)
    recs["flags"][:, ::7] &= ~np.uint8(8)                 # without VALID: no reward, the tally still counts
    labels = ((np.arange(T) * 7919) % G).astype(np.uint8)
    engine.record_groups_upload(labels, G)
    model = gf.rec_model(recs, labels, G)
    engine.rollouts_upload(recs)
    check(engine.score(C, 2, source=apo.SRC_ROLLOUTS, groups=True).groups, model)
    check(engine.score_host_records(recs, 2, groups=True).groups, model)
    check(engine.score(C, 2, source=apo.SRC_ROLLOUTS, recip=True, groups=True).groups, gf.rec_model(recs, labels, G, recip=True))
    p16 = apo.pack16(recs)
    model16 = gf.rec_model(orc.unpack16(p16), labels, G)
    engine.rollouts16_upload(p16)
    check(engine.score(C, 2, source=apo.SRC_ROLLOUTS, groups=True).groups, model16)
    check(engine.score_host_records(p16, 2, groups=True).groups, model16)
    C2, T2 = 64, 300_001                                  # across the window boundary (R: 131 072, R16: 262 144 records)
    big = orc.gen_records(0x5EED6E04, orc.STREAM_ROLLOUT, 0, C2, 0, T2, 300, 8)
    labels2 = (np.arange(T2) % 3).astype(np.uint8)
    engine.record_groups_upload(labels2, 3)
    got = engine.score_host_records(big, 2, groups=True).groups
    for c in (0, C2 - 1):
        check([got[c]], gf.rec_model(big[c:c + 1], labels2, 3))
    assert bytes(engine.score_host_records(apo.pack16(big), 2, groups=True).groups) == bytes(got)


def test_windows_sessions_and_chunks(engine, orc, apo):
    C, T, G = 6, 40_000, 5
    dims = orc.gen_dims(0x5EED6E05, 0, C, 0, T, 300, 8)
    labels = ((np.arange(T) // 1000) % G).astype(np.uint8)
    engine.record_groups_upload(labels, G)
    engine.dims_upload(dims)
    for first, count in ((4, 10_000), (36, 0), (1000, 33)):          # windows off the 32-grid
        end = T if count == 0 else first + count
        check(engine.score(C, 1, first=first, count=count, groups=True).groups, window_model(dims, labels, G, first, end))
    whole = gf.model(dims, labels, G)
    engine.score_begin(C)                                              # candidate chunks, windows in reverse order
    for c0 in (3, 0):
        engine.dims_upload(dims[c0:c0 + 3])
        engine.score_accumulate(c0, first=20_004, count=0, groups=True)
        engine.score_accumulate(c0, first=0, count=20_004, groups=True)
    check(engine.score_finish(C, 2, groups=True).groups, whole)
    check(engine.score_finish(C, 2, groups=True).groups, whole)        # finish may be repeated
    engine.dims_upload(dims)                                           # the same window twice counts twice
    engine.score_begin(C)
    engine.score_accumulate(0, first=0, count=4096, groups=True)
    engine.score_accumulate(0, first=0, count=4096, groups=True)
    fr, ok = final_rewards(dims[:, :4096])
    two = gf.group_model(np.tile(fr, 2), np.tile(ok, 2), np.tile(gf.dims_tally(dims[:, :4096]), 2), np.tile(labels[:4096], 2), G)
    check(engine.score_finish(C, 1, groups=True).groups, two)
    pc, pd, book, d2book = apo.packed_encode_host(dims)               # resident Form T windows
    tl, th, tbook = apo.tuple_encode_host(pc, pd)
    engine.tuples_upload(tl, th, tbook, book, d2book)
    engine.score_begin(C)
    engine.score_accumulate(0, source=apo.SRC_TUPLES, first=8200, count=0, groups=True)
    engine.score_accumulate(0, source=apo.SRC_TUPLES, first=8, count=8192, groups=True)
    check(engine.score_finish(C, 1, groups=True).groups, window_model(dims, labels, G, 8, T))


def test_refusals(engine, orc, apo):
    C, T = 4, 5000
    dims = orc.gen_dims(0x5EED6E06, 0, C, 0, T, 300, 8)
    engine.dims_upload(dims)

    def code(fn, *a, **kw):
        with pytest.raises(apo.ApoError) as ei:
            fn(*a, **kw)
        return ei.value.code

    engine.record_groups_upload(np.zeros(0, np.uint8))                 # released
    assert code(engine.score, C, 1, groups=True) == -3                 # no labels
    assert code(engine.candidate_groups, 0, C, 1) == -3                # a failed call leaves no groups behind
    labels = (np.arange(T) % 3).astype(np.uint8)
    assert code(engine.record_groups_upload, labels, 0) == -1
    assert code(engine.record_groups_upload, labels, 65) == -1
    assert code(engine.record_groups_upload, labels, 2) == -1          # a label >= G
    engine.record_groups_upload(labels[:T - 1], 3)
    assert code(engine.score, C, 1, groups=True) == -1                 # the last position is past the labels
    check(engine.score(C, 1, count=T - 1, groups=True).groups, window_model(dims, labels, 3, 0, T - 1))
    assert code(engine.record_groups_upload, np.full(T, 7, np.uint8), 4) == -1
    check(engine.score(C, 1, count=T - 1, groups=True).groups, window_model(dims, labels, 3, 0, T - 1))   # the labels stayed
    engine.record_groups_upload(labels, 3)
    assert code(engine.candidate_groups, 0, C, 2) == -1                # not the G the call scored with
    assert code(engine.candidate_groups, C - 1, 2) == -1
    engine.score(C, 1)
    assert code(engine.candidate_groups, 0, C) == -3                   # the last call did not set the flag
    engine.score_begin(C)                                              # a mixed session
    engine.score_accumulate(0, first=0, count=2000, groups=True)
    engine.score_accumulate(0, first=2000, count=0)
    assert code(engine.score_finish, C, 1, groups=True) == -3
    assert code(engine.candidate_groups, 0, C) == -3
    engine.score_begin(C)                                              # labels uploaded again during a flagged session
    engine.score_accumulate(0, first=0, count=2000, groups=True)
    engine.record_groups_upload((np.arange(T) % 5).astype(np.uint8), 5)
    engine.score_accumulate(0, first=2000, count=0, groups=True)
    assert code(engine.score_finish, C, 1, groups=True) == -3
    engine.record_groups_upload(labels[:100], 3)
    assert code(engine.score_host, dims, 1, groups=True) == -1         # the streamed call's T is past the labels
    res = engine.score(C, 1, count=64, groups=True)
    check(res.groups, window_model(dims, labels, 3, 0, 64))


def test_flags_together_and_flag_clear_unchanged(engine, orc, apo):
    C, T, G = 5, 30_000, 6
    recs = orc.gen_records(0x5EED6E07, orc.STREAM_ROLLOUT, 0, C, 0, T, 300, 8)
    corpus = orc.gen_records(0x5EED6E07, orc.STREAM_CORPUS, 0, 1, 0, 3000, 300, 8).reshape(-1)
    labels = ((np.arange(T) // 37) % G).astype(np.uint8)
    engine.record_groups_upload(labels, G)
    engine.rollouts_upload(recs)
    engine.corpus_upload(corpus)
    model = gf.rec_model(recs, labels, G)

    def call(**kw):
        r = engine.score(C, 3, source=apo.SRC_ROLLOUTS, corpus=True, **kw)
        return r, (r.scores.tobytes(), r.counts.tobytes(), r.topk.tobytes(), bytes(r.report))

    plain, key = call()
    alone = {f: bytes(getattr(call(**{f: True})[0], a)) for f, a in
             (("candidates", "candidates"), ("candidate_corpus", "candidate_corpus"), ("extremes", "extremes"))}
    for mask in range(16):
        flags = {f: bool(mask >> i & 1) for i, f in enumerate(("candidates", "candidate_corpus", "extremes", "groups"))}
        r, k = call(**flags)
        assert k == key, flags
        if flags["groups"]:
            check(r.groups, model)
        else:
            assert r.groups is None
        for f, a in (("candidates", "candidates"), ("candidate_corpus", "candidate_corpus"), ("extremes", "extremes")):
            if flags[f]:
                assert bytes(getattr(r, a)) == alone[f], flags
    r, _ = call(groups=True)
    assert r.timing.launches == plain.timing.launches + 2                 # the pass and its conversion
    again, k2 = call()
    assert k2 == key and again.timing.launches == plain.timing.launches


GRID_SCRIPT = textwrap.dedent("""
    import sys, numpy as np
    sys.path.insert(0, {root!r})
    import importlib
    apo = importlib.import_module("senweaver-ide_b200")
    e = apo.Engine(0)
    dims, labels = np.load({path!r}), np.load({lpath!r})
    e.record_groups_upload(labels, 64)
    e.set_tuning(0x10)
    e.dims_upload(dims)
    out = e.score(dims.shape[0], 1, groups=True).groups
    e.close()
    sys.stdout.write(bytes(out).hex())
""")


def test_forced_grids(orc, apo, tmp_path):
    """1 ... 7 CTAs (APO_K1_GRID, read once per process: a subprocess each): rows span several warps and flushes"""
    T = 3 * 1024 + 40
    d = orc.gen_dims(0x5EED6E08, 0, 3, 0, T, 300, 4)
    labels = np.where(np.arange(T) < 2000, np.arange(T) % 64, (np.arange(T) // 500) % 64).astype(np.uint8)
    path, lpath = str(tmp_path / "dims.npy"), str(tmp_path / "labels.npy")
    np.save(path, d)
    np.save(lpath, labels)
    outs = set()
    for g in range(1, 8):
        env = dict(os.environ, APO_K1_GRID=str(g))
        script = GRID_SCRIPT.format(root=ROOT, path=path, lpath=lpath)
        r = subprocess.run([sys.executable, "-c", script], env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr
        outs.add(r.stdout)
    assert len(outs) == 1
    got = ((importlib.import_module("senweaver-ide_b200.engine").GroupScore * 64) * 3).from_buffer_copy(bytes.fromhex(outs.pop()))
    check(got, gf.model(d, labels, 64))


def test_custom_zero_and_recip_weights(engine, orc, apo):
    C, T, G = 4, 20_000, 5
    dims = orc.gen_dims(0x5EED6E09, 0, C, 0, T, 300, 8)
    dims[:, ::5, 1:3] = np.nan
    labels = ((np.arange(T) * 31) % G).astype(np.uint8)
    engine.record_groups_upload(labels, G)
    try:
        for w in (np.array([0.0, 0.3, 0.0, 0.1, 0.2, 0.0, 0.1, 0.2, 0.1]), np.array([0.0] * 8 + [1.0]), np.linspace(0.05, 0.45, 9)):
            engine.set_weights(w)
            for tune in (0x10, 0):
                engine.set_tuning(tune)
                engine.dims_upload(dims)
                for recip in (False, True):
                    check(engine.score(C, 2, recip=recip, groups=True).groups, gf.model(dims, labels, G, w, recip))
    finally:
        engine.set_tuning(0)
        engine.set_weights(orc.weights())


def test_many_candidates_g64(engine, orc):
    C, T, G = 16384, 96, 64
    dims = orc.gen_dims(0x5EED6E0A, 0, C, 0, T, 300, 8)
    dims[:, ::3, :] = np.nan
    labels = (np.arange(T) % G).astype(np.uint8)
    engine.record_groups_upload(labels, G)
    engine.dims_upload(dims)
    res = engine.score(C, 16, groups=True)
    check(res.groups, gf.model(dims, labels, G))
    assert [sum(s.withReward for s in row) for row in res.groups] == [int(n) for n in res.counts]


def test_full_size_256x5M_against_the_generator(engine, orc, apo):
    """config 3 (256 x 5 M, 46 GB Form D resident) through its default route, byte-equal to K1; spread rows against the
    generator's rows"""
    seed, C, T, G = 0x5EED0003, 256, 5_000_000, 5
    labels = ((np.arange(T) // 4099) % G).astype(np.uint8)
    engine.record_groups_upload(labels, G)
    engine.dims_generate(seed, 0, C, 0, T, 300)
    res = engine.score(C, 4, groups=True)
    engine.set_tuning(0x10)
    try:
        res_k1 = engine.score(C, 4, groups=True)
    finally:
        engine.set_tuning(0)
    assert bytes(res_k1.groups) == bytes(res.groups)
    assert [sum(s.withReward for s in row) for row in res.groups] == [int(n) for n in res.counts]
    for c in (0, 85, 170, 255):
        check([res.groups[c]], gf.model(orc.gen_dims(seed, c, 1, 0, T, 300, 16), labels, G))


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
            e.record_groups_upload(np.zeros(2 * T, np.uint8), 1)
            e.dims_generate(0x5EED6E0B, 0, C, rank * T, T, 300)
            try:
                e.score(C, 1, groups=True)
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
