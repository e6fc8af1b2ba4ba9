"""Form D with its Form W copy (-m gpu).  When no coded dimension of a loaded Form D tensor takes more than 15 values (true for
every tensor TCS:668-763 produces), the copy built at load is one 8-byte word per evaluation (eight 4-bit codes, fp32
tool_success_rate) instead of the 14-byte Form Q planes, and K1q reads it.  Every result must equal the oracle's integers and
the TUNE_NO_TWIN run (K1 on the fp32 tensor) of the same engine; a profiler record shows which K1q instantiation ran (its
last template argument: true = Form W)."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import k1_fixtures as kf
from test_gpu_dims_twin import categorical, kernels, same, same_bits

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
NAN = np.float32(np.nan)
TILE = 20 * 32 * 8                      # K1q's tile on Form W (and Form Q's default): 20 consumer warps x 8 evaluations


def layout_of(names):
    """'W', 'Q' or 'K1': what the scoring kernel in a profiler record read"""
    m = re.search(r"k_reward9q<([^>]*)>", names)
    if m:
        return "W" if m.group(1).split(",")[-1].strip() == "true" else "Q"
    m = re.search(r"k_reward9qI(\w*?)EEvNS_8KqParams", names)           # not demangled
    if m:
        return "W" if m.group(1).endswith("Lb1E") else "Q"
    assert "k_reward9<36" in names or "k_reward9ILi36E" in names, names
    return "K1"


def reads(fn):
    return layout_of(kernels(fn))


def exact(engine, apo, C, call, want, layout="W"):
    """call() reads `layout`; its integers are `want` and those of the TUNE_NO_TWIN run (K1), with the same results"""
    engine.set_tuning(0)
    if layout:
        assert reads(call) == layout
    r = call()
    p = engine.debug_partials(C)
    assert p == want
    engine.set_tuning(apo.TUNE_NO_TWIN)
    try:
        assert reads(call) == "K1"
        r1 = call()
        assert engine.debug_partials(C) == p and same(r, r1)
    finally:
        engine.set_tuning(0)
    return r


def masks_dims(T=512 * 8):
    """[3][T][9]: every presence mask of the nine dimensions, coded values +0.0 / -0.0 / 0.5 / -1.0 / 1.0 (distinct codes),
    tool_success_rate 0.0, -0.0, 0.25 or -0.75 where present"""
    t = np.arange(T)
    d = np.empty((3, T, 9), np.float32)
    levels = np.array([0.0, -0.0, 0.5, -1.0, 1.0], np.float32)
    d2 = np.array([0.0, -0.0, 0.25, -0.75], np.float32)
    for c in range(3):
        for i in range(9):
            d[c, :, i] = levels[(t * 7 + i + 3 * c) % 5]
            d[c, ((t + 37 * c) % 512 >> i) & 1 == 0, i] = NAN
        p2 = ~np.isnan(d[c, :, 2])
        d[c, p2, 2] = d2[((t // 512) + c) % 4][p2]
    return d


def levels_dims(nvals, C=3, T=40_000, seed=71):
    """categorical dims whose dimension 4 takes exactly `nvals` values (the others a handful)"""
    d = categorical(seed, C, T)
    rng = np.random.default_rng(seed)
    vals = np.linspace(-1, 1, nvals).astype(np.float32)
    d[:, :, 4] = vals[rng.integers(0, nvals, (C, T))]
    d[:, :nvals, 4] = vals                                                        # every value occurs
    return d


@pytest.mark.parametrize("load", ["upload", "generate"])
def test_generated_dims_read_the_word_copy(engine, orc, apo, load):
    seed, C, T = 0x5EED7020, 6, 50_001
    dims = orc.gen_dims(seed, 2, C, 300, T, 400, 8)
    if load == "upload":
        engine.dims_upload(dims)
    else:
        engine.dims_generate(seed, 2, C, 300, T, 400)
    assert engine.dims_layout() == 1
    assert same_bits(engine.dims_download(3, 1000, 700), dims[3, 1000:1700])
    recs = orc.gen_records(seed, orc.STREAM_CORPUS, 0, 1, 0, 20_000, 300, 8).reshape(-1)
    engine.corpus_upload(recs)
    r = exact(engine, apo, C, lambda: engine.score(C, 2, corpus=True), orc.score_dims_fx(dims))
    assert r.timing.launches == 1 and r.report.bad == orc.report(recs).bad
    for first, count, layout in ((8000, 20_003, "W"), (4004, 10_000, "K1"), (T - 1, 0, "W"), (TILE, TILE + 8, "W")):
        end = first + count if count else T
        exact(engine, apo, C, lambda: engine.score(C, 1, first=first, count=count), orc.score_dims_fx(dims[:, first:end]), layout)
    for recip in (False, True):
        exact(engine, apo, C, lambda: engine.score(C, C, recip=recip), kf.fx_model(dims, recip=True) if recip else orc.score_dims_fx(dims))

    def session():
        engine.score_begin(C + 2)
        engine.score_accumulate(2, count=24_000)
        engine.score_accumulate(2, first=24_000, count=12_004)                  # the cut at 36_004 is off the grid: K1
        engine.score_accumulate(2, first=36_004)
        return engine.score_finish(C + 2, 3, corpus=True)

    names = kernels(session)
    assert layout_of(names) == "W" and ("k_reward9<36" in names or "k_reward9ILi36E" in names)
    sums, counts = orc.score_dims_fx(dims)
    exact(engine, apo, C + 2, session, ([0, 0] + list(sums), [0, 0] + list(counts)), layout=None)


def test_fifteen_values_give_the_word_copy_sixteen_form_q(engine, orc, apo):
    for nvals, layout in ((15, "W"), (16, "Q")):
        dims = levels_dims(nvals)
        engine.dims_upload(dims)
        exact(engine, apo, 3, lambda: engine.score(3, 2), orc.score_dims_fx(dims), layout)
        exact(engine, apo, 3, lambda: engine.score(3, 2, candidates=True), orc.score_dims_fx(dims), layout)


def test_every_presence_mask_and_signed_zeros(engine, orc, apo):
    dims = masks_dims()
    engine.dims_upload(dims)
    for recip in (False, True):
        want = kf.fx_model(dims, recip=True) if recip else orc.score_dims_fx(dims)
        exact(engine, apo, 3, lambda: engine.score(3, 3, recip=recip, candidates=True), want)
    w = np.array([0.3, 0.1, 0.05, 0.05, 0.1, 0.1, 0.1, 0.1, 0.1])                  # total weight with an all-ones significand
    wz = np.array([0.0, 0.4, 0.05, 0.0, 0.1, 0.1, 0.15, 0.1, 0.1])                 # zero weights: all-null masks exist
    try:
        for weights in (w, wz):
            engine.set_weights(weights)
            exact(engine, apo, 3, lambda: engine.score(3, 3), orc.score_dims_fx(dims, w=weights))
    finally:
        engine.set_weights(orc.weights())


@pytest.mark.parametrize("which", ["extreme", "ties", "edges"])
def test_k1_fixtures(engine, apo, which):
    if which == "extreme":
        dims = kf.extreme_dims()
    elif which == "ties":
        dims = kf.tie_dims()
    else:
        rows = [kf.shape_dims(1, T, seed=k)[0] for k, T in enumerate(kf.t_edges(TILE))]
        T = max(len(r) for r in rows)
        dims = np.stack([np.concatenate([r, np.full((T - len(r), 9), NAN, np.float32)]) for r in rows])
    C = dims.shape[0]
    engine.dims_upload(dims)
    layout = "W" if all(len(np.unique(dims[:, :, i][~np.isnan(dims[:, :, i])].view(np.uint32))) <= 15
                        for i in (0, 1, 3, 4, 5, 6, 7, 8)) else "Q"
    for recip in (False, True):
        exact(engine, apo, C, lambda: engine.score(C, C, recip=recip), kf.fx_model(dims, recip=recip), layout)


def test_huge_sums(engine, apo):
    dims = kf.huge_dims()
    engine.dims_upload(dims)
    exact(engine, apo, 2, lambda: engine.score(2, 2), kf.fx_model(dims))


GRID_SCRIPT = r"""
import importlib, json, sys
sys.path[:0] = [sys.argv[1], sys.argv[2]]
import k1_fixtures as kf
apo = importlib.import_module("senweaver-ide_b200")
e = apo.Engine(0)
out = {}
for C, T in ((3, 2 * 5120 + 1), (2, 5 * 5120 - 8), (300, 7)):
    e.dims_upload(kf.shape_dims(C, T, seed=C))
    e.score(C, 1)
    s, n = e.debug_partials(C)
    out[f"{C}/{T}"] = [[str(x) for x in s], n]
e.close()
print(json.dumps(out))
"""


@pytest.mark.parametrize("grid", [1, 2, 3, 7])
def test_forced_grid(apo, grid):
    """APO_K1_GRID (read once per process) forces K1q on the word copy down to `grid` CTAs"""
    env = dict(os.environ, APO_K1_GRID=str(grid))
    p = subprocess.run([sys.executable, "-c", GRID_SCRIPT, ROOT, HERE], env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-3000:]
    got = json.loads(p.stdout.strip().splitlines()[-1])
    for C, T in ((3, 2 * TILE + 1), (2, 5 * TILE - 8), (300, 7)):
        s, n = got[f"{C}/{T}"]
        assert ([int(x) for x in s], n) == tuple(kf.oracle_fx(kf.shape_dims(C, T, seed=C))), (C, T)


def test_domain_refusal(engine, orc, apo):
    dims = orc.gen_dims(0x5EED7021, 0, 3, 0, 20_000, 300, 8)
    for v in (512.0, -513.0):
        big = dims.copy()
        big[1, 77] = NAN
        big[1, 77, 0] = v
        engine.dims_upload(big)

        def refused():
            with pytest.raises(apo.ApoError):
                engine.score(3, 1)

        assert reads(refused) == "W"
    engine.dims_upload(dims)
    exact(engine, apo, 3, lambda: engine.score(3, 1), orc.score_dims_fx(dims))


def test_streamed_calls_compact_and_breakdown(engine, orc, apo):
    seed, C, T = 0x5EED7022, 4, 40_000
    dims = orc.gen_dims(seed, 0, C, 0, T, 300, 8)
    exp = orc.score_dims_fx(dims)
    other = orc.gen_dims(0x5EED7011, 40, 3, 0, 30_000, 900, 8)                    # another codebook
    exp_other = orc.score_dims_fx(other)
    engine.dims_upload(dims)
    exact(engine, apo, C, lambda: engine.score(C, 2, candidates=True), exp)
    q8, d2, li, book = apo.compact_encode_host(other, nthreads=4)
    engine.score_host_compact(q8, d2, li, book, 1)
    assert engine.debug_partials(3) == exp_other
    exact(engine, apo, C, lambda: engine.score(C, 2), exp)
    pc, pd, pbook, d2book = apo.packed_encode_host(other, nthreads=4)
    engine.score_host_packed(pc, pd, pbook, d2book, 1)
    assert engine.debug_partials(3) == exp_other
    exact(engine, apo, C, lambda: engine.score(C, 2), exp)
    # apo_dims_compact with the word copy held: the copy goes, the fp32 tensor is transcoded to the planes
    q8, d2, li, book = apo.compact_encode_host(dims, nthreads=4)
    engine.dims_compact()
    assert engine.dims_layout() == 2
    assert np.array_equal(engine.dims_codebook(), book)
    a, b, l = engine.dims_compact_download(2, 0, T)
    assert np.array_equal(a, q8[2]) and np.array_equal(b.view(np.uint32), d2[2].view(np.uint32)) and np.array_equal(l, li[2])
    assert reads(lambda: engine.score(C, 2)) == "Q"
    engine.score(C, 2)
    assert engine.debug_partials(C) == exp


def round_up(x, m):
    return (x + m - 1) // m * m


@pytest.mark.parametrize("room", ["form_q_only", "none"])
def test_room_for_form_q_only_and_for_none(orc, apo, room):
    """the word copy is packed beside the Form Q planes: with room for the planes but not for both (4 GiB headroom) the
    Form Q copy is kept; with room for neither, no copy"""
    import torch
    seed, C, T = 0x5EED7023, 32, 1_000_000
    n = C * round_up(T, 32)
    exp = orc.score_dims_fx(orc.gen_dims(seed, 0, C, 0, T, 300, 8))
    e = apo.Engine(0)
    filler = None
    try:
        e.dims_generate(seed, 0, C, 0, T, 300)
        assert reads(lambda: e.score(C, 4)) == "W"
        free = torch.cuda.mem_get_info()[0] + 8 * n                             # at the next load's check, the word copy released
        target = 18 * n + (4 << 30) if room == "form_q_only" else 14 * n + (3 << 30)
        filler = torch.empty(free - target, dtype=torch.uint8, device="cuda")
        e.dims_generate(seed, 0, C, 0, T, 300)
        assert reads(lambda: e.score(C, 4)) == ("Q" if room == "form_q_only" else "K1")
        e.score(C, 4)
        assert e.debug_partials(C) == exp
    finally:
        del filler
        torch.cuda.empty_cache()
        e.close()
