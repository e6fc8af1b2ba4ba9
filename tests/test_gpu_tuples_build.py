"""Form T built on the device (apo_dims_tuples, csrc/apo_tuple.cu k_tb_*) on the H100 (-m gpu).

Everything is exact.  The dictionary, codebooks and index planes equal, byte for byte, what the host chain makes of the same
tensor (apo_packed_encode_host -> apo_tuple_encode_host), from the Form W copy (apo_dims_upload, apo_dims_generate) and from
a Form Q layout (apo_dims_upload_compact, apo_dims_compact after a load), for generated and hand-built tensors and for forced
small grids.  Scoring the result (source APO_SRC_TUPLES) gives the integers, scores, top-K, breakdown and corpus report of
source APO_SRC_DIMS on the same engine."""
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN = np.float32("nan")
APO_E_ARG, APO_E_STATE, APO_E_NOMEM = -1, -3, -4
TUPLES_MAX = 0xFFFFFF
SEED = 0x5EED7300


def host_chain(apo, dims, cap=TUPLES_MAX):
    pc, pd, book, d2book = apo.packed_encode_host(dims)
    tl, th, tb = apo.tuple_encode_host(pc, pd, cap=cap)
    return tl, th, tb, book, d2book


def device_form_t(engine, C, T):
    tb, book, d2book = engine.tuples_book()
    tl, th = np.empty((C, T), np.uint16), np.empty((C, T), np.uint8)
    for c in range(C):
        tl[c], th[c] = engine.tuples_download(c, 0, T)
    return tl, th, tb, book, d2book


def assert_host_bytes(engine, apo, dims, n):
    C, T, _ = dims.shape
    want = host_chain(apo, dims)
    got = device_form_t(engine, C, T)
    assert n == want[2][0].size
    for w, g in zip(want[:2], got[:2]):
        assert w.tobytes() == g.tobytes()
    assert want[2][0].tobytes() == got[2][0].tobytes() and want[2][1].tobytes() == got[2][1].tobytes()
    assert want[3].tobytes() == got[3].tobytes() and want[4].tobytes() == got[4].tobytes()
    return got


def load(engine, kind, dims):
    if kind == "upload":
        engine.dims_upload(dims)
    elif kind == "upload_compact":
        engine.dims_upload_compact(dims)
    elif kind == "compact":
        engine.dims_upload(dims)
        engine.dims_compact()
    else:
        raise ValueError(kind)


def same_scoring(engine, apo, C, **kw):
    """SRC_TUPLES and SRC_DIMS on the same engine: partials, scores, counts, top-K, breakdown and report"""
    K = kw.pop("K", min(C, 4))
    a = engine.score(C, K, source=apo.SRC_DIMS, **kw)
    pa = engine.debug_partials(C)
    b = engine.score(C, K, source=apo.SRC_TUPLES, **kw)
    assert engine.debug_partials(C) == pa
    assert a.scores.tobytes() == b.scores.tobytes() and a.counts.tobytes() == b.counts.tobytes()
    assert np.array_equal(a.topk, b.topk)
    if kw.get("candidates"):
        assert bytes(a.candidates) == bytes(b.candidates)
    if kw.get("corpus"):
        assert bytes(a.report) == bytes(b.report)
    return pa


def expect_error(code, fn):
    with pytest.raises(Exception) as ex:
        fn()
    assert getattr(ex.value, "code", None) == code, str(ex.value)
    return ex.value


# ---------------------------------------------------------------- byte equality with the host chain
SHAPES = [(1, 1), (1, 7), (3, 1000), (17, 4099), (64, 1_000_003)]


@pytest.mark.parametrize("kind", ["upload", "generate", "upload_compact", "compact"])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"{c}x{t}" for c, t in SHAPES])
def test_bytes_equal_the_host_chain(engine, orc, apo, kind, shape):
    C, T = shape
    dims = orc.gen_dims(SEED, 3, C, 100, T, 300, 8)
    if kind == "generate":
        engine.dims_generate(SEED, 3, C, 100, T, 300)
    else:
        load(engine, kind, dims)
    n = engine.dims_tuples()
    assert_host_bytes(engine, apo, dims, n)
    same_scoring(engine, apo, C)


# ---------------------------------------------------------------- hand-built tensors
def cat_dims(C, T, seed=5):
    """categorical dims with a handful of values per coded dimension and 40 tool_success_rate values"""
    rng = np.random.default_rng(seed)
    lv = np.array([-1.0, -0.5, 0.0, 0.3, 0.8, 1.0], np.float32)
    d = lv[rng.integers(0, 6, (C, T, 9))]
    d[:, :, 2] = np.linspace(-1, 1, 40).astype(np.float32)[rng.integers(0, 40, (C, T))]
    d[rng.random((C, T, 9)) < 0.1] = NAN
    return d


def distinct_dims(T, C=1):
    """evaluation i (row-major) is distinct for i < 4000 * 11^3: d2 from 4000 values, dims 0, 1, 3 from base-11 digits"""
    i = np.arange(C * T).reshape(C, T)
    d = np.full((C, T, 9), 0.5, np.float32)
    v = np.linspace(-1, 1, 11).astype(np.float32)
    d[:, :, 2] = np.linspace(-1, 1, 4000).astype(np.float32)[i % 4000]
    d[:, :, 0] = v[(i // 4000) % 11]
    d[:, :, 1] = v[(i // 44000) % 11]
    d[:, :, 3] = v[(i // 484000) % 11]
    return d


def check_tensor(engine, apo, dims, kinds=("upload", "upload_compact")):
    for kind in kinds:
        load(engine, kind, dims)
        n = engine.dims_tuples()
        assert_host_bytes(engine, apo, dims, n)
        same_scoring(engine, apo, dims.shape[0])
    return n


def test_one_distinct_evaluation(engine, apo):
    d = np.tile(np.array([1, 0.5, 0.25, 1, -0.3, 0, 1, 0.3, 0.8], np.float32), (5, 3001, 1))
    assert check_tensor(engine, apo, d) == 1
    tl, th = engine.tuples_download(4, 0, 3001)
    assert not tl.any() and not th.any()


def test_all_null_rows(engine, apo):
    d = cat_dims(6, 2077)
    d[1] = NAN
    d[4, :1000] = NAN
    check_tensor(engine, apo, d)


def test_signed_zeros(engine, apo):
    d = cat_dims(3, 4100)
    d[:, ::3, 2] = np.float32(-0.0)
    d[:, 1::3, 2] = np.float32(0.0)
    d[:, ::5, 4] = np.float32(-0.0)
    d[:, 2::5, 4] = np.float32(0.0)
    check_tensor(engine, apo, d)


@pytest.mark.parametrize("nd2", [4095, 4096])
def test_d2_values(engine, apo, nd2):
    d = cat_dims(2, 9000)
    vals = np.linspace(-1, 1, nd2).astype(np.float32)
    assert np.unique(vals).size == nd2
    d[:, :, 2] = vals[np.arange(2 * 9000).reshape(2, 9000) % nd2]
    if nd2 == 4095:
        check_tensor(engine, apo, d)
    else:
        for kind in ("upload", "upload_compact"):
            load(engine, kind, d)
            expect_error(APO_E_STATE, engine.dims_tuples)
            expect_error(APO_E_STATE, lambda: engine.score(2, 1, source=apo.SRC_TUPLES))


@pytest.mark.parametrize("nvals", [15, 16])
def test_coded_values(engine, apo, nvals):
    d = cat_dims(3, 5000)
    vals = np.linspace(-1, 1, nvals).astype(np.float32)
    d[:, :, 4] = vals[np.arange(3 * 5000).reshape(3, 5000) % nvals]
    if nvals == 15:
        check_tensor(engine, apo, d, ("upload", "upload_compact", "compact"))
    else:
        for kind in ("upload", "upload_compact"):            # a Form Q copy, then a Form Q layout
            load(engine, kind, d)
            e = expect_error(APO_E_STATE, engine.dims_tuples)
            assert "16 or more" in str(e)


def test_equal_frequencies_across_ctas(engine, apo):
    """600 keys, each 2000 times, interleaved so that every CTA holds a different partial count of each: the order comes from
    the key ties alone"""
    k = 600
    base = distinct_dims(k)[0]
    perm = np.random.default_rng(9).permutation(k * 2000) % k
    d = base[perm].reshape(8, k * 250, 9)
    assert check_tensor(engine, apo, d) == k


def test_one_dominant_key_and_singletons(engine, apo):
    T = 400_000
    d = np.tile(np.array([1, 0.5, 0.25, 1, -0.3, 0, 1, 0.3, 0.8], np.float32), (2, T, 1))
    single = distinct_dims(60_000)[0]
    pos = np.random.default_rng(3).choice(2 * T, 60_000, replace=False)
    d.reshape(-1, 9)[pos] = single
    assert check_tensor(engine, apo, d, ("upload",)) == 60_001


@pytest.mark.parametrize("T,past", [(29_003, 24_576), (77_011, 65_536), (1_230_007, 1 << 20)])
def test_large_dictionaries(engine, apo, T, past):
    d = distinct_dims(T)
    d[0, 1::7] = d[0, ::7][: d[0, 1::7].shape[0]]                           # some repeats: counts 1 and 2
    n = check_tensor(engine, apo, d, ("upload",))
    assert n > past
    if n > 65_536:
        _, th = engine.tuples_download(0, 0, T)
        assert th.any()


def test_cap(engine, apo):
    d = distinct_dims(5000, C=2)                                              # 10 000 distinct evaluations
    engine.dims_upload(d)
    assert engine.dims_tuples(10_000) == 10_000
    e = expect_error(APO_E_STATE, lambda: engine.dims_tuples(9_999))
    assert e.n_tuples > 9_999
    expect_error(APO_E_STATE, lambda: engine.score(2, 1, source=apo.SRC_TUPLES))
    e = expect_error(APO_E_STATE, lambda: engine.dims_tuples(0))
    assert e.n_tuples > 0
    assert engine.dims_tuples(TUPLES_MAX + 5) == 10_000                        # clamped


# ---------------------------------------------------------------- grid independence
GRID_SCRIPT = r"""
import hashlib, importlib, sys
sys.path.insert(0, {root!r})
apo = importlib.import_module("senweaver-ide_b200")
e = apo.Engine(0)
e.dims_generate({seed}, 0, 9, 0, 70001, 300)
n = e.dims_tuples()
h = hashlib.sha256()
(pc, pd), cb, d2 = e.tuples_book()
for a in (pc, pd, cb, d2):
    h.update(a.tobytes())
for c in range(9):
    for a in e.tuples_download(c, 0, 70001):
        h.update(a.tobytes())
print(n, h.hexdigest())
"""


def test_grid_independence(apo):
    script = GRID_SCRIPT.format(root=ROOT, seed=SEED + 1)
    out = []
    for grid in (None, "1", "7"):
        env = dict(os.environ)
        env.pop("APO_K1_GRID", None)
        if grid:
            env["APO_K1_GRID"] = grid
        r = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, env=env, cwd=ROOT, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        out.append(r.stdout.split()[-2:])
    assert out[0] == out[1] == out[2]


# ---------------------------------------------------------------- scoring equivalence
@pytest.fixture()
def built(engine, orc, apo):
    C, T = 6, 50_001
    engine.set_weights(np.array([0.25, 0.18, 0.12, 0.08, 0.05, 0.05, 0.08, 0.08, 0.11]))
    engine.dims_generate(SEED + 2, 0, C, 0, T, 400)
    engine.dims_tuples()
    yield C, T
    engine.set_weights(np.array([0.25, 0.18, 0.12, 0.08, 0.05, 0.05, 0.08, 0.08, 0.11]))


def test_windows(engine, apo, built):
    C, T = built
    for first, count in ((0, 0), (8, 16_000), (40_000, 0), (24_000, 8)):
        same_scoring(engine, apo, C, first=first, count=count)


def test_session(engine, apo, built):
    C, T = built
    parts = []
    for src in (apo.SRC_DIMS, apo.SRC_TUPLES):
        engine.score_begin(C + 1)
        engine.score_accumulate(1, source=src, count=16_000)
        engine.score_accumulate(1, source=src, first=16_000, count=8_008)
        engine.score_accumulate(1, source=src, first=24_008)
        r = engine.score_finish(C + 1, 3)
        parts.append((engine.debug_partials(C + 1), r.scores.tobytes(), r.topk.tolist()))
    assert parts[0] == parts[1]


def test_recip_weights_candidates_corpus(engine, apo, built):
    C, T = built
    same_scoring(engine, apo, C, recip=True)
    engine.set_weights(np.array([0.3, 0.0, 0.7, 0.1, 0.0, 0.2, 0.05, 0.0, 0.4]))
    same_scoring(engine, apo, C)
    engine.set_weights(np.zeros(9))
    p = same_scoring(engine, apo, C)
    assert p[1] == [0] * C
    engine.set_weights(np.array([0.25, 0.18, 0.12, 0.08, 0.05, 0.05, 0.08, 0.08, 0.11]))
    same_scoring(engine, apo, C, candidates=True)
    engine.corpus_generate(SEED + 3, 0, 20_000, 300)
    same_scoring(engine, apo, C, corpus=True)
    engine.corpus_upload(np.zeros(0, apo.RECORD_DTYPE))


# ---------------------------------------------------------------- state
def test_state(engine, orc, apo):
    C, T = 4, 30_011
    dims = orc.gen_dims(SEED + 4, 0, C, 0, T, 300, 8)
    engine.dims_upload(dims)
    want = orc.score_dims_fx(dims)
    engine.score(C, 2)
    assert engine.debug_partials(C) == want
    n = engine.dims_tuples()
    engine.score(C, 2)                                                        # the dims' own scoring is unchanged
    assert engine.debug_partials(C) == want
    assert engine.dims_download(2, 100, 50).tobytes() == dims[2, 100:150].tobytes()
    other = orc.gen_dims(SEED + 5, 0, 3, 0, 999, 300, 8)
    engine.dims_upload(other)                                                 # later loads leave the tuples alone
    engine.score(C, 2, source=apo.SRC_TUPLES)
    assert engine.debug_partials(C) == want
    assert engine.tuples_book()[0][0].size == n
    # uploaded tuples replace them and round-trip through the exports
    tl, th, tb, book, d2b = host_chain(apo, other)
    engine.tuples_upload(tl, th, tb, book, d2b)
    got = device_form_t(engine, 3, 999)
    assert got[0].tobytes() == tl.tobytes() and got[1].tobytes() == th.tobytes()
    assert got[2][0].tobytes() == tb[0].tobytes() and got[2][1].tobytes() == tb[1].tobytes()
    assert got[3].tobytes() == book.tobytes() and got[4].tobytes() == d2b.tobytes()
    engine.score(3, 1, source=apo.SRC_TUPLES)
    assert engine.debug_partials(3) == orc.score_dims_fx(other)


def test_refusals(apo):
    import ctypes as C
    e = apo.Engine(0)
    try:
        expect_error(APO_E_STATE, e.dims_tuples)                              # nothing loaded
        expect_error(APO_E_STATE, e.tuples_book)
        expect_error(APO_E_STATE, lambda: e.tuples_download(0, 0, 1))
        d = cat_dims(3, 3000)
        e.set_tuning(apo.TUNE_NO_TWIN)
        e.dims_upload(d)
        assert "apo_dims_compact" in str(expect_error(APO_E_STATE, e.dims_tuples))
        e.set_tuning(0)
        e.dims_upload(d)
        e.set_tuning(apo.TUNE_NO_TWIN)                                        # a copy held but not to be read
        expect_error(APO_E_STATE, e.dims_tuples)
        e.set_tuning(0)
        import torch
        buf = torch.from_numpy(np.ascontiguousarray(d)).cuda()
        e.dims_attach(buf.data_ptr(), 3, 3000, 3000)
        assert "apo_dims_compact" in str(expect_error(APO_E_STATE, e.dims_tuples))
        e.dims_compact()                                                      # the way out
        assert e.dims_tuples() > 0
        del buf
        L, h = e._L, e._h
        assert L.apo_dims_tuples(h, 100, None) == APO_E_ARG
        assert L.apo_dims_tuples(None, 100, None) == APO_E_ARG
        tl, th = np.empty(10, np.uint16), np.empty(10, np.uint8)
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        assert L.apo_tuples_download(h, None, p(th), 0, 0, 1) == APO_E_ARG
        assert L.apo_tuples_download(h, p(tl), None, 0, 0, 1) == APO_E_ARG
        assert L.apo_tuples_download(h, p(tl), p(th), 3, 0, 1) == APO_E_ARG
        assert L.apo_tuples_download(h, p(tl), p(th), 0, 2995, 6) == APO_E_ARG
        assert L.apo_tuples_download(h, p(tl), p(th), 0, 2995, 5) == 0
        assert L.apo_tuples_download(h, p(tl), p(th), 0, (1 << 64) - 1, 2) == APO_E_ARG
        n = C.c_uint32(0)
        cb, d2 = np.empty(2048, np.uint32), np.empty(4096, np.uint32)
        full = e.tuples_book()[0][0].size
        pc, pd = np.empty(full, np.uint32), np.empty(full, np.uint16)
        assert L.apo_tuples_book(h, p(pc), p(pd), full - 1, p(cb), p(d2), C.addressof(n)) == APO_E_ARG and n.value == full
        assert L.apo_tuples_book(h, p(pc), p(pd), full, None, p(d2), C.addressof(n)) == APO_E_ARG
        assert L.apo_tuples_book(h, p(pc), p(pd), full, p(cb), None, C.addressof(n)) == APO_E_ARG
        assert L.apo_tuples_book(h, None, p(pd), full, p(cb), p(d2), C.addressof(n)) == APO_E_ARG
        assert L.apo_tuples_book(h, p(pc), p(pd), full, p(cb), p(d2), None) == APO_E_ARG
        assert L.apo_tuples_book(h, p(pc), p(pd), full, p(cb), p(d2), C.addressof(n)) == 0
    finally:
        e.close()


def round_up(x, m):
    return (x + m - 1) // m * m


def test_build_that_fits_only_without_the_copy(orc, apo):
    """the build's allocations release the Form W copy it would read: APO_E_NOMEM, no Form T, the dims still score exactly"""
    import torch
    C, T, cap = 32, 1_000_000, 1 << 20
    exp = orc.score_dims_fx(orc.gen_dims(SEED + 6, 0, C, 0, T, 300, 8))
    copy = C * round_up(T, 32) * 8
    slots = 1024
    while slots < 2 * (cap + 1):
        slots *= 2
    need = C * round_up(T, 64) * 3 + cap * 6 + 4096 * 4 + slots * 16 + cap * 16
    e = apo.Engine(0)
    filler = None
    try:
        e.dims_generate(SEED + 6, 0, C, 0, T, 300)
        free = torch.cuda.mem_get_info()[0]
        leave = need - copy // 2                                               # < need <= leave + copy
        assert free > leave + (1 << 30)
        filler = torch.empty(free - leave, dtype=torch.uint8, device="cuda")
        expect_error(APO_E_NOMEM, lambda: e.dims_tuples(cap))
        expect_error(APO_E_STATE, lambda: e.score(C, 2, source=apo.SRC_TUPLES))
        e.score(C, 2)
        assert e.debug_partials(C) == exp
    finally:
        del filler
        torch.cuda.empty_cache()
        e.close()


def test_full_size(apo):
    """256 x 5 M on bench.py's generator and seed: 293 177 distinct evaluations, and the integers of SRC_TUPLES equal SRC_DIMS.

    The tensor is generated straight into the Form Q layout (apo_dims_generate_compact: the same generator, the same
    evaluations), 18 GB instead of the 46 GB fp32 tensor plus the copies apo_dims_generate builds beside it, so the test does
    not depend on the device memory other engines of the test process still hold.  The Form W source is checked byte for byte
    against the host chain at 64 x 1 M above; at this size it is measured by examples/tuples_build.py."""
    bench_seed = 0x5EED0003
    C, T = 256, 5_000_000
    e = apo.Engine(0)
    try:
        e.dims_generate_compact(bench_seed, 0, C, 0, T, 300)
        assert e.dims_layout() == 2
        n = e.dims_tuples()
        a = e.score(C, 8)
        pa = e.debug_partials(C)
        b = e.score(C, 8, source=apo.SRC_TUPLES)
        assert e.debug_partials(C) == pa
        assert a.scores.tobytes() == b.scores.tobytes() and np.array_equal(a.topk, b.topk)
        print(f"n_tuples at 256 x 5M: {n}")
        assert n == 293_177
    finally:
        e.close()
