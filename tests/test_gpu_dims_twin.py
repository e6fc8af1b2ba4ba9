"""Form D with its Form Q copy (-m gpu).  apo_dims_upload / apo_dims_generate also build a lossless 14 B/eval copy of a
categorical tensor, and resident Form D calls with variant 0 and a window on the 8-evaluation grid read it through K1q;
every other call reads the fp32 tensor through K1.  Every result must equal the oracle's integers and the TUNE_NO_TWIN run
(K1 on the fp32 tensor) of the same engine; a profiler record of one call shows which scoring kernel ran."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

def kernels(fn, tries=3):
    """the names of the CUDA kernels fn launched, from a torch.profiler record.  fn is a scoring call, so it launches a
    k_reward9* kernel; now and then a record holds the call's cudaLaunchKernel and no kernel at all (see
    test_gpu_dims_tuple_copy.kernels).  Such a record says nothing about the route, so fn() is profiled again."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    for _ in range(tries):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = " ".join(ev.name for ev in prof.events())
        if "k_reward9" in names:
            break
    return names


def reads(engine, fn):
    """'K1q' or 'K1': the scoring kernel fn ran (k_reward9q, or k_reward9<36, ...> demangled or not)"""
    names = kernels(fn)
    q, d = "k_reward9q" in names, "k_reward9<36" in names or "k_reward9ILi36E" in names
    assert q != d, names
    return "K1q" if q else "K1"


def same(a, b):
    ok = np.array_equal(a.scores, b.scores) and np.array_equal(a.counts, b.counts) and np.array_equal(a.topk, b.topk)
    if a.candidates is not None:
        ok &= memoryview(a.candidates).tobytes() == memoryview(b.candidates).tobytes()
    return ok


def with_and_without(engine, apo, C, call):
    """call() reading the copy where it applies, then with TUNE_NO_TWIN (K1 on the fp32 tensor): the same results and
    integers.  Returns the integers."""
    engine.set_tuning(0)
    r = call()
    p = engine.debug_partials(C)
    engine.set_tuning(apo.TUNE_NO_TWIN)
    try:
        assert reads(engine, call) == "K1"
        r1 = call()
        assert engine.debug_partials(C) == p and same(r, r1)
    finally:
        engine.set_tuning(0)
    return p


def categorical(seed, C, T):
    """hand-built categorical dims: every presence mask, +-0.0, free-form fp32 tool_success_rate"""
    rng = np.random.default_rng(seed)
    levels = np.array([-1.0, -0.8, -0.5, -0.3, -0.2, 0.0, -0.0, 0.3, 0.5, 0.8, 1.0], np.float32)
    dims = levels[rng.integers(0, len(levels), (C, T, 9))]
    dims[:, :, 2] = rng.uniform(-1, 1, (C, T)).astype(np.float32)
    dims[rng.random(dims.shape) < 0.3] = np.nan
    dims[C - 1, : T // 2] = np.nan
    return dims


def same_bits(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    nan = np.isnan(a)
    return np.array_equal(nan, np.isnan(b)) and np.array_equal(a[~nan].view(np.uint32), b[~nan].view(np.uint32))


@pytest.mark.parametrize("load", ["upload", "generate"])
def test_windows_and_sessions_on_and_off_the_grid(engine, orc, apo, load):
    seed, C, T = 0x5EED7010, 6, 50_001
    dims = orc.gen_dims(seed, 2, C, 300, T, 400, 8)
    if load == "upload":
        engine.dims_upload(dims)
    else:
        engine.dims_generate(seed, 2, C, 300, T, 400)
    assert engine.dims_layout() == 1
    assert same_bits(engine.dims_download(3, 1000, 700), dims[3, 1000:1700])      # the fp32 tensor stays loaded
    recs = orc.gen_records(seed, orc.STREAM_CORPUS, 0, 1, 0, 20_000, 300, 8).reshape(-1)
    engine.corpus_upload(recs)
    assert reads(engine, lambda: engine.score(C, 2, corpus=True)) == "K1q"
    r = engine.score(C, 2, corpus=True)
    assert r.timing.launches == 1 and r.report.bad == orc.report(recs).bad       # corpus scan and tail ride on K1q
    assert with_and_without(engine, apo, C, lambda: engine.score(C, 2, corpus=True)) == orc.score_dims_fx(dims)
    for first, count, kernel in ((8000, 20_003, "K1q"), (4004, 10_000, "K1"), (T - 1, 0, "K1q"), (T - 5, 0, "K1")):
        call = lambda: engine.score(C, 1, first=first, count=count)
        assert reads(engine, call) == kernel, (first, count)
        end = first + count if count else T
        assert with_and_without(engine, apo, C, call) == orc.score_dims_fx(dims[:, first:end]), (first, count)
    # a session whose accumulates read the copy and the fp32 tensor: the cut at 12_004 is off the grid
    exp = orc.score_dims_fx(dims)

    def session():
        engine.score_begin(C + 2)
        engine.score_accumulate(2, count=24_000)
        engine.score_accumulate(2, first=24_000, count=12_004)
        engine.score_accumulate(2, first=36_004)
        return engine.score_finish(C + 2, 3, corpus=True)

    sums, counts = with_and_without(engine, apo, C + 2, session)
    assert counts[:2] == [0, 0] and (sums[2:], counts[2:]) == exp


@pytest.mark.parametrize("recip", [False, True])
def test_variants_and_recip(engine, orc, apo, recip):
    C, T = 5, 30_000
    dims = categorical(41, C, T)
    engine.dims_upload(dims)
    for variant in range(5):
        call = lambda: engine.score(C, C, variant=variant, recip=recip)
        assert reads(engine, call) == ("K1q" if variant == 0 else "K1"), variant
        p = with_and_without(engine, apo, C, call)
        if not recip:
            assert p == orc.score_dims_fx(dims), variant
    # the fixed-point domain flag: a finalReward beyond 512 is refused on both paths
    big = dims.copy()
    big[1, 77] = np.nan
    big[1, 77, 0] = 1e6
    engine.dims_upload(big)
    for tuning in (0, apo.TUNE_NO_TWIN):
        engine.set_tuning(tuning)
        try:
            with pytest.raises(apo.ApoError):
                engine.score(C, 1, recip=recip)
        finally:
            engine.set_tuning(0)


def test_weights_set_after_the_load(engine, orc, apo):
    C, T = 4, 20_000
    dims = categorical(43, C, T)
    engine.dims_upload(dims)
    engine.score(C, 1)
    w = np.array([0.3, 0.1, 0.05, 0.05, 0.1, 0.1, 0.1, 0.1, 0.1])              # total weight with an all-ones significand
    wz = np.array([0.0, 0.4, 0.05, 0.0, 0.1, 0.1, 0.15, 0.1, 0.1])             # zero weights: all-null masks exist
    try:
        for weights in (w, wz, orc.weights()):
            engine.set_weights(weights)
            assert reads(engine, lambda: engine.score(C, C)) == "K1q"
            assert with_and_without(engine, apo, C, lambda: engine.score(C, C)) == orc.score_dims_fx(dims, w=weights)
    finally:
        engine.set_weights(orc.weights())


def test_streamed_form_q_and_p_between_resident_calls(engine, orc, apo):
    """a streamed Form Q / P call swaps in its own codebook's tables; the copy gets its own back"""
    C, T = 4, 40_000
    dims = categorical(47, C, T)
    exp = orc.score_dims_fx(dims)
    other = orc.gen_dims(0x5EED7011, 40, 3, 0, 30_000, 900, 8)                 # another codebook
    exp_other = orc.score_dims_fx(other)
    engine.dims_upload(dims)
    engine.score(C, 2)
    assert engine.debug_partials(C) == exp
    q8, d2, li, book = apo.compact_encode_host(other, nthreads=4)
    engine.score_host_compact(q8, d2, li, book, 1)
    assert engine.debug_partials(3) == exp_other
    assert reads(engine, lambda: engine.score(C, 2)) == "K1q"
    assert with_and_without(engine, apo, C, lambda: engine.score(C, 2)) == exp
    pc, pd, pbook, d2book = apo.packed_encode_host(other, nthreads=4)
    engine.score_host_packed(pc, pd, pbook, d2book, 1)
    assert engine.debug_partials(3) == exp_other
    engine.score(C, 2)
    assert engine.debug_partials(C) == exp


def test_candidate_breakdown(engine, orc, apo):
    seed, C, T = 0x5EED7012, 5, 40_000
    engine.dims_generate(seed, 0, C, 0, T, 300)
    exp = orc.score_dims_fx(orc.gen_dims(seed, 0, C, 0, T, 300, 8))
    assert reads(engine, lambda: engine.score(C, 2, candidates=True)) == "K1q"
    assert with_and_without(engine, apo, C, lambda: engine.score(C, 2, candidates=True)) == exp

    def session():
        engine.score_begin(C)
        engine.score_accumulate(0, count=16_004, candidates=True)               # K1q
        engine.score_accumulate(0, first=16_004, candidates=True)               # off the grid: K1
        return engine.score_finish(C, 2, candidates=True)

    assert with_and_without(engine, apo, C, session) == exp


def test_dims_compact_after_the_load(engine, orc, apo):
    C, T = 4, 25_000
    dims = categorical(53, C, T)
    exp = orc.score_dims_fx(dims)
    q8, d2, li, book = apo.compact_encode_host(dims, nthreads=4)
    for tuning in (0, apo.TUNE_NO_TWIN):                                        # with the copy held, and without one
        engine.set_tuning(tuning)
        try:
            engine.dims_upload(dims)
            engine.dims_compact()
        finally:
            engine.set_tuning(0)
        assert engine.dims_layout() == 2
        assert np.array_equal(engine.dims_codebook(), book)
        a, b, l = engine.dims_compact_download(2, 0, T)
        assert np.array_equal(a, q8[2]) and np.array_equal(b.view(np.uint32), d2[2].view(np.uint32)) and np.array_equal(l, li[2])
        assert same_bits(engine.dims_download(1, 0, T), dims[1])
        engine.score(C, 2)
        assert engine.debug_partials(C) == exp
        with pytest.raises(apo.ApoError):
            engine.score(C, 1, first=4, count=100)                              # a compact tensor refuses windows off the grid


def test_non_categorical_dims_stay_on_k1(engine, orc, apo):
    rng = np.random.default_rng(59)
    dims = rng.uniform(-1, 1, (3, 4000, 9)).astype(np.float32)                  # > 255 distinct values per dimension
    engine.dims_upload(dims)                                                     # no error, no error text
    assert b"categorical" not in (engine._L.apo_last_error(engine._h) or b"")
    assert engine.dims_layout() == 1
    assert reads(engine, lambda: engine.score(3, 1)) == "K1"
    engine.score(3, 1)
    assert engine.debug_partials(3) == orc.score_dims_fx(dims)


def round_up(x, m):
    return (x + m - 1) // m * m


def test_no_copy_without_room(orc, apo):
    """with less than 4 GiB free beside the copy none is built, and the results stay exact"""
    import torch
    seed, C, T = 0x5EED7013, 32, 1_000_000
    exp = orc.score_dims_fx(orc.gen_dims(seed, 0, C, 0, T, 300, 8))
    e = apo.Engine(0)
    filler = None
    try:
        e.dims_generate(seed, 0, C, 0, T, 300)
        assert reads(e, lambda: e.score(C, 4)) == "K1q"
        free = torch.cuda.mem_get_info()[0]                                      # with the copy held
        assert free > (3 << 30)
        filler = torch.empty(free - (3 << 30), dtype=torch.uint8, device="cuda")
        e.dims_generate(seed, 0, C, 0, T, 300)                                   # about the copy + 3 GiB free at the check
        assert reads(e, lambda: e.score(C, 4)) == "K1"
        e.score(C, 4)
        assert e.debug_partials(C) == exp
    finally:
        del filler
        torch.cuda.empty_cache()
        e.close()


def test_allocation_that_fits_only_without_the_copy(orc, apo):
    """a rollouts load that fits only once the copy is released succeeds, and both sources keep scoring exactly"""
    import torch
    seed, C, T = 0x5EED7014, 32, 1_000_000
    exp = orc.score_dims_fx(orc.gen_dims(seed, 0, C, 0, T, 300, 8))
    copy = C * round_up(T, 32) * 14
    Cr, Tr = 8, 2_000_000
    rbytes = Cr * round_up(Tr, 4) * 32
    e = apo.Engine(0)
    filler = None
    try:
        e.dims_generate(seed, 0, C, 0, T, 300)
        assert reads(e, lambda: e.score(C, 4)) == "K1q"
        free = torch.cuda.mem_get_info()[0]
        leave = rbytes - copy // 2                                               # < rbytes <= leave + copy
        assert free > leave + (1 << 30)
        filler = torch.empty(free - leave, dtype=torch.uint8, device="cuda")
        e.rollouts_generate(seed, 0, Cr, 0, Tr, 300)
        e.score(Cr, 2, source=apo.SRC_ROLLOUTS)
        s, n = e.debug_partials(Cr)
        for c in (0, Cr - 1):
            rs, rn = orc.score_records_fx(orc.gen_records(seed, orc.STREAM_ROLLOUT, c, 1, 0, Tr, 300, 8))
            assert (s[c], n[c]) == (rs[0], rn[0])
        assert reads(e, lambda: e.score(C, 4)) == "K1"                          # the copy is gone: K1 on the fp32 tensor
        e.score(C, 4)
        assert e.debug_partials(C) == exp
    finally:
        del filler
        torch.cuda.empty_cache()
        e.close()
