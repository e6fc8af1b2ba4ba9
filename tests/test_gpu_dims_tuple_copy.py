"""Form D with its Form T copy (-m gpu).  apo_dims_upload / apo_dims_generate build a Form T copy (3 B/eval dictionary
indices) beside the Form W / Q copy of a large tensor, and resident Form D calls with variant 0 and a window on the
8-evaluation grid read it through K1t, with table values computed at load / apo_set_weights (no k_tuple_values per call).
TUNE_TWIN_T builds the copy for the small tensors here.  Every result must equal the oracle's integers (the numpy model for
recip) and those of the TUNE_NO_TWIN_T (K1q on the Form W copy) and TUNE_NO_TWIN (K1 on the fp32 tensor) runs of the same
engine; a profiler record of one call shows which scoring kernel ran."""
import os
import sys
from importlib import import_module

import numpy as np
import pytest

import k1_fixtures as kf
from test_gpu_dims_twin import categorical, same
from test_gpu_dims_twin import kernels as profiled_kernels
from test_gpu_dims_word import layout_of as word_layout

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def forced(engine, apo):
    """loads in these tests build the Form T copy whatever their size; the shared engine gets its default back"""
    engine.set_tuning(apo.TUNE_TWIN_T)
    yield
    engine.set_tuning(0)


SCORING = ("k_reward9t", "k_reward9q", "k_reward9<36", "k_reward9ILi36E")


def kernels(fn, tries=3):
    """kernel names of fn() from a torch.profiler record.  Every call here launches a scoring kernel, but about one record
    in a thousand holds the cudaLaunchKernel of a call and no kernel at all (measured on an H100 with single-launch calls,
    whatever the route): such a record says nothing about the route, so fn() is profiled again"""
    for _ in range(tries):
        names = profiled_kernels(fn)
        if any(k in names for k in SCORING):
            break
    return names


def layout_of(names):
    """'T' (K1t on the copy, without a per-call k_tuple_values), 'W', 'Q' or 'K1'"""
    if "k_reward9t" in names:
        assert "k_tuple_values" not in names, names
        return "T"
    return word_layout(names)


def reads(fn):
    return layout_of(kernels(fn))


def exact(engine, apo, C, call, want, layout="T"):
    """call() reads `layout`; its integers are `want` (None: not checked) and those of the TUNE_NO_TWIN_T run (the Form W /
    Q copy) and the TUNE_NO_TWIN run (K1), with the same results.  The routes of those two settings are pinned by
    test_gpu_dims_word / test_gpu_dims_twin and test_route_flags here; only the route under test is profiled."""
    engine.set_tuning(apo.TUNE_TWIN_T)
    call()                                       # the first call with recip set computes the copy's values for it, once
    if layout:
        assert reads(call) == layout
    r = call()
    p = engine.debug_partials(C)
    if want is not None:
        assert p == want
    try:
        for flags in (apo.TUNE_NO_TWIN_T, apo.TUNE_NO_TWIN):
            engine.set_tuning(flags)
            r1 = call()
            assert engine.debug_partials(C) == p and same(r, r1)
    finally:
        engine.set_tuning(apo.TUNE_TWIN_T)
    return r


def cat_dims(seed, C, T):
    """categorical dims (presence masks of every kind, +-0.0) drawn from 5000 distinct evaluations whose tool_success_rate
    takes 200 values: Form T can index them and K1t's shared-memory head holds them all"""
    pool = categorical(seed, 1, 5000)[0]
    rng = np.random.default_rng(seed + 1)
    p2 = ~np.isnan(pool[:, 2])
    pool[p2, 2] = rng.uniform(-1, 1, 200).astype(np.float32)[rng.integers(0, 200, int(p2.sum()))]
    d = pool[rng.integers(0, len(pool), (C, T))]
    d[C - 1, : T // 2] = np.nan
    return d


@pytest.mark.parametrize("load", ["upload", "generate"])
def test_windows_recip_beam_widths_corpus(engine, orc, apo, load):
    seed, C, T = 0x5EED7030, 6, 50_001
    dims = orc.gen_dims(seed, 2, C, 300, T, 400, 8)
    if load == "upload":
        engine.dims_upload(dims)
    else:
        engine.dims_generate(seed, 2, C, 300, T, 400)
    assert engine.dims_layout() == 1
    recs = orc.gen_records(seed, orc.STREAM_CORPUS, 0, 1, 0, 20_000, 300, 8).reshape(-1)
    engine.corpus_upload(recs)
    exp = orc.score_dims_fx(dims)
    r = exact(engine, apo, C, lambda: engine.score(C, 2, corpus=True), exp)
    assert r.timing.launches == 2 and r.report.bad == orc.report(recs).bad        # K1t, then the corpus scan with the tail
    for first, count, layout in ((8000, 20_003, "T"), (4004, 10_000, "K1"), (T - 1, 0, "T"), (8192, 8200, "T"), (T - 5, 0, "K1")):
        end = first + count if count else T
        exact(engine, apo, C, lambda: engine.score(C, 1, first=first, count=count), orc.score_dims_fx(dims[:, first:end]), layout)
    for recip in (False, True, False):                                          # the recip values are computed once, then kept
        exact(engine, apo, C, lambda: engine.score(C, C, recip=recip), kf.fx_model(dims, recip=True) if recip else exp)
    for K in range(1, C + 1):
        exact(engine, apo, C, lambda: engine.score(C, K, corpus=True), exp)
    exact(engine, apo, C, lambda: engine.score(C, 2, candidates=True), exp)
    for variant in range(1, 5):
        exact(engine, apo, C, lambda: engine.score(C, 2, variant=variant), exp, "K1")


def test_route_flags(engine, orc, apo):
    """with the copy held: K1t by default, K1q on the Form W copy with TUNE_NO_TWIN_T, K1 with TUNE_NO_TWIN"""
    C, T = 4, 30_000
    dims = orc.gen_dims(0x5EED7038, 0, C, 0, T, 300, 8)
    engine.dims_upload(dims)
    for flags, layout in ((apo.TUNE_TWIN_T, "T"), (apo.TUNE_NO_TWIN_T, "W"), (apo.TUNE_NO_TWIN, "K1"), (0, "T")):
        engine.set_tuning(flags)
        assert reads(lambda: engine.score(C, 2)) == layout, flags
        engine.score(C, 2)
        assert engine.debug_partials(C) == orc.score_dims_fx(dims)


def test_sessions_mix_the_copy_and_k1(engine, orc, apo):
    seed, C, T = 0x5EED7031, 5, 40_000
    dims = orc.gen_dims(seed, 0, C, 0, T, 300, 8)
    engine.dims_upload(dims)
    sums, counts = orc.score_dims_fx(dims)

    def session(cand=False):
        engine.score_begin(C + 2)
        engine.score_accumulate(2, count=24_000, candidates=cand)                # K1t
        engine.score_accumulate(2, first=24_000, count=12_004, candidates=cand)  # K1t; the cut at 36_004 is off the grid
        engine.score_accumulate(2, first=36_004, candidates=cand)                # K1
        return engine.score_finish(C + 2, 3, corpus=True, candidates=cand)

    names = kernels(session)
    assert "k_reward9t" in names and "k_tuple_values" not in names and ("k_reward9<36" in names or "k_reward9ILi36E" in names)
    want = ([0, 0] + list(sums), [0, 0] + list(counts))
    exact(engine, apo, C + 2, session, want, layout=None)
    exact(engine, apo, C + 2, lambda: session(True), want, layout=None)


def test_weights_set_after_the_load(engine, orc, apo):
    C, T = 4, 20_000
    dims = cat_dims(43, C, T)
    engine.dims_upload(dims)
    w = np.array([0.3, 0.1, 0.05, 0.05, 0.1, 0.1, 0.1, 0.1, 0.1])              # total weight with an all-ones significand
    wz = np.array([0.0, 0.4, 0.05, 0.0, 0.1, 0.1, 0.15, 0.1, 0.1])             # zero weights: all-null masks exist
    try:
        for weights in (w, wz, orc.weights()):
            engine.set_weights(weights)
            exact(engine, apo, C, lambda: engine.score(C, C), orc.score_dims_fx(dims, w=weights))
            exact(engine, apo, C, lambda: engine.score(C, C, recip=True), kf.fx_model(dims, w=weights, recip=True))
    finally:
        engine.set_weights(orc.weights())


def test_values_outside_the_copy_domain(engine, orc, apo):
    """a finalReward in [2, 512) is exact on the Form W copy, which such calls read; beyond 512 every route refuses"""
    C, T = 3, 30_000
    dims = cat_dims(47, C, T)
    big = dims.copy()
    big[1, 77] = np.nan
    big[1, 77, 0] = 5.0
    engine.dims_upload(big)
    exact(engine, apo, C, lambda: engine.score(C, 2), orc.score_dims_fx(big), "W")
    exact(engine, apo, C, lambda: engine.score(C, 2, recip=True), kf.fx_model(big, recip=True), "W")
    big[1, 77, 0] = 1e6
    engine.dims_upload(big)
    for flags in (apo.TUNE_TWIN_T, apo.TUNE_NO_TWIN_T, apo.TUNE_NO_TWIN):
        engine.set_tuning(flags)
        for recip in (False, True):
            with pytest.raises(apo.ApoError):
                engine.score(C, 1, recip=recip)
    engine.set_tuning(apo.TUNE_TWIN_T)
    engine.dims_upload(dims)                                                     # the handle stays usable and exact
    exact(engine, apo, C, lambda: engine.score(C, 2), orc.score_dims_fx(dims))


def test_no_copy_past_its_limits(engine, orc, apo):
    """more than 2^20 distinct evaluations, a flat distribution (K1t's shared-memory head would serve a quarter of the
    reads), or a tool_success_rate with more than 4095 values: the Form W copy, no error"""
    rng = np.random.default_rng(53)
    C, T = 2, 700_000
    levels = np.array([-1.0, -0.8, -0.5, -0.3, -0.2, 0.0, 0.3, 0.5, 0.8, 1.0], np.float32)
    d = levels[rng.integers(0, len(levels), (C, T, 9))]
    d[:, :, 2] = levels[rng.integers(0, len(levels), (C, T))]                   # ~1.4 M distinct of 10^9
    engine.dims_upload(d)                                                       # no error
    exact(engine, apo, C, lambda: engine.score(C, 1), orc.score_dims_fx(d), "W")
    pool = np.unique(levels[rng.integers(0, len(levels), (110_000, 9))], axis=0)[:100_000]
    flat = pool[rng.integers(0, len(pool), (C, 200_000))]                       # the 24576 most frequent: ~1/4 of the reads
    engine.dims_upload(flat)
    exact(engine, apo, C, lambda: engine.score(C, 1), orc.score_dims_fx(flat), "W")
    free = categorical(59, 3, 5000)                                             # fp32 tool_success_rate: ~10^4 values
    engine.dims_upload(free)
    exact(engine, apo, 3, lambda: engine.score(3, 1), orc.score_dims_fx(free), "W")


def test_the_copy_is_not_resident_form_t(orc, apo):
    C, T = 3, 20_000
    dims = orc.gen_dims(0x5EED7037, 0, C, 0, T, 300, 8)
    e = apo.Engine(0)
    try:
        e.set_tuning(apo.TUNE_TWIN_T)
        e.dims_upload(dims)
        assert reads(lambda: e.score(C, 1)) == "T"
        with pytest.raises(apo.ApoError, match="no tuples loaded"):
            e.score(C, 1, source=apo.SRC_TUPLES)
        with pytest.raises(apo.ApoError):
            e.tuples_book()
    finally:
        e.close()


def test_tuples_state_is_independent(engine, orc, apo):
    C, T = 4, 30_011
    dims = orc.gen_dims(0x5EED7032, 0, C, 0, T, 300, 8)
    other = orc.gen_dims(0x5EED7033, 0, 3, 0, 999, 300, 8)
    want, want_other = orc.score_dims_fx(dims), orc.score_dims_fx(other)
    engine.dims_upload(other)
    engine.dims_tuples()                                                        # resident Form T of `other`
    engine.dims_upload(dims)                                                    # a copy of `dims` beside it
    engine.score(3, 1, source=apo.SRC_TUPLES)
    assert engine.debug_partials(3) == want_other
    exact(engine, apo, C, lambda: engine.score(C, 2), want)
    n = engine.dims_tuples()                                                    # Form T of `dims`: the copy stays as it was
    assert engine.tuples_book()[0][0].size == n
    engine.score(C, 2, source=apo.SRC_TUPLES)
    assert engine.debug_partials(C) == want
    exact(engine, apo, C, lambda: engine.score(C, 2), want)
    pc, pd, book, d2book = apo.packed_encode_host(other, nthreads=2)
    tl, th, tbook = apo.tuple_encode_host(pc, pd, nthreads=2)
    engine.tuples_upload(tl, th, tbook, book, d2book)                           # an uploaded Form T replaces the resident one
    exact(engine, apo, C, lambda: engine.score(C, 2), want)
    engine.score(3, 1, source=apo.SRC_TUPLES)
    assert engine.debug_partials(3) == want_other


def test_compact_attach_and_new_loads_drop_the_copy(engine, orc, apo):
    import torch
    C, T = 4, 25_000
    dims = cat_dims(61, C, T)
    exp = orc.score_dims_fx(dims)
    engine.dims_upload(dims)
    exact(engine, apo, C, lambda: engine.score(C, 2), exp)
    engine.dims_compact()
    assert engine.dims_layout() == 2
    assert reads(lambda: engine.score(C, 2)) == "Q"                            # the compact layout: K1q on Form Q
    engine.score(C, 2)
    assert engine.debug_partials(C) == exp
    engine.dims_upload(dims)
    exact(engine, apo, C, lambda: engine.score(C, 2), exp)
    buf = torch.from_numpy(np.ascontiguousarray(dims)).cuda()
    engine.dims_attach(buf.data_ptr(), C, T, T)
    assert reads(lambda: engine.score(C, 2)) == "K1"
    engine.score(C, 2)
    assert engine.debug_partials(C) == exp
    del buf
    engine.set_tuning(0)
    engine.dims_upload(dims)                                                    # below the size rule: the Form W copy only
    assert reads(lambda: engine.score(C, 2)) == "W"
    engine.set_tuning(apo.TUNE_TWIN_T)
    engine.dims_upload(dims)
    assert reads(lambda: engine.score(C, 2)) == "T"


def round_up(x, m):
    return (x + m - 1) // m * m


def test_allocation_that_fits_only_without_the_copies(orc, apo):
    """a rollouts load that fits only once the Form W and Form T copies are released succeeds, and both sources stay exact"""
    import torch
    seed, C, T = 0x5EED7034, 32, 1_000_000
    exp = orc.score_dims_fx(orc.gen_dims(seed, 0, C, 0, T, 300, 8))
    copies = C * round_up(T, 32) * 8 + C * round_up(T, 64) * 3
    Cr, Tr = 8, 2_000_000
    rbytes = Cr * round_up(Tr, 4) * 32
    e = apo.Engine(0)
    filler = None
    try:
        e.set_tuning(apo.TUNE_TWIN_T)
        e.dims_generate(seed, 0, C, 0, T, 300)
        assert reads(lambda: e.score(C, 4)) == "T"
        free = torch.cuda.mem_get_info()[0]
        leave = rbytes - copies // 2                                             # < rbytes <= leave + copies
        assert free > leave + (1 << 30)
        filler = torch.empty(free - leave, dtype=torch.uint8, device="cuda")
        e.rollouts_generate(seed, 0, Cr, 0, Tr, 300)
        e.score(Cr, 2, source=apo.SRC_ROLLOUTS)
        s, n = e.debug_partials(Cr)
        for c in (0, Cr - 1):
            rs, rn = orc.score_records_fx(orc.gen_records(seed, orc.STREAM_ROLLOUT, c, 1, 0, Tr, 300, 8))
            assert (s[c], n[c]) == (rs[0], rn[0])
        assert reads(lambda: e.score(C, 4)) == "K1"                              # the copies are gone: K1 on the fp32 tensor
        e.score(C, 4)
        assert e.debug_partials(C) == exp
    finally:
        del filler
        torch.cuda.empty_cache()
        e.close()


def test_size_rule(engine, apo):
    """without TUNE_TWIN_T the copy is built from 2^26 evaluations on"""
    seed, C = 0x5EED7035, 64
    engine.set_tuning(0)
    for T, layout in (((1 << 20) - 1, "W"), (1 << 20, "T")):
        engine.dims_generate(seed, 0, C, 0, T, 300)
        assert C * T < (1 << 26) if layout == "W" else C * T >= (1 << 26)
        exact(engine, apo, C, lambda: engine.score(C, 8), None, layout)
        engine.set_tuning(0)
    engine.set_tuning(apo.TUNE_NO_TWIN_T)
    engine.dims_generate(seed, 0, C, 0, 1 << 20, 300)                           # nothing built: nothing to read either
    engine.set_tuning(0)
    assert reads(lambda: engine.score(C, 8)) == "W"


def worker(rank, world, port_path, out_dir, C, T):
    import torch
    sys.path.insert(0, ROOT)
    pkg = import_module("senweaver-ide_b200")
    torch.cuda.set_device(rank)
    eng = pkg.Engine(rank)
    eng.comm_init(world, rank, open(port_path, "rb").read())
    eng.set_tuning(pkg.TUNE_TWIN_T)                 # every rank its own dictionary over its shard
    first, last = pkg.sharding.shard_range(T, world, rank)
    eng.dims_generate(0x5EED7036, 0, C, first, last - first, 300)
    eng.corpus_generate(0x5EED7036, first, last - first, 300)
    names = kernels(lambda: eng.score(C, 3, corpus=True))
    for _ in range(3):
        res = eng.score(C, 3, corpus=True)
    sums, counts = eng.debug_partials(C)
    np.savez(os.path.join(out_dir, f"r{rank}.npz"), scores=res.scores, topk=res.topk, sums=np.array([str(s) for s in sums]),
             bad=np.array([res.report.bad]), t=np.array(["k_reward9t" in names and "k_tuple_values" not in names]))
    eng.close()


def test_world_2_peer_join(tmp_path, engine, apo):
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    C, T = 8, 400_003
    uid = tmp_path / "uid.bin"
    uid.write_bytes(apo.Engine.comm_unique_id())
    mp.spawn(worker, args=(2, str(uid), str(tmp_path), C, T), nprocs=2, join=True)
    engine.set_tuning(apo.TUNE_NO_TWIN)
    engine.dims_generate(0x5EED7036, 0, C, 0, T, 300)
    engine.corpus_generate(0x5EED7036, 0, T, 300)
    ref = engine.score(C, 3, corpus=True)
    rsums, _ = engine.debug_partials(C)
    for r in range(2):
        z = np.load(tmp_path / f"r{r}.npz")
        assert z["t"][0] and [int(s) for s in z["sums"]] == rsums
        assert np.array_equal(z["scores"], ref.scores) and np.array_equal(z["topk"], ref.topk) and z["bad"][0] == ref.report.bad
