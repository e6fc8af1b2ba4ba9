"""The Form T copy read from its 16-bit plane (-m gpu).  When at most 1/64 of a copy's evaluations have a dictionary index
of 2^16 or more, the load lists them (the exceptions) and resident Form D calls run K1t2 (k_reward9t2): 2 B per
evaluation from tl, then a correction of the listed evaluations inside the same launch.  The tensors here hold 65 536
frequent evaluations, each at least twice (ranks below 2^16), and rare ones, each once (ranks 2^16 and up: exactly the
exceptions), placed to give every layout of the list: positions 0 and T-1, a run longer than a warp, a block of 8192
exceptions, a row without and a row of only exceptions, and a row whose net count correction is negative under weights
that leave the rare evaluations uncounted.  Every result must equal the oracle's integers (the numpy model for recip) and
those of the TUNE_NO_TWIN_T2 (K1t on tl / th), TUNE_NO_TWIN_T (K1q) and TUNE_NO_TWIN (K1) runs of the same engine.
Whether a call reads the list follows from whether the load built one (apo_debug_twin_t_list).  The module takes no
torch.profiler records (test_gpu_dims_tuple_copy names the kernel of the copy's route): on an H100, a process's profiler
records lost their kernels once its first profiler session lay a few tens of seconds back."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

import k1_fixtures as kf
from test_gpu_dims_twin import same

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
XBLOCK = 8192
NF = 1 << 16
C, T = 128, 20_009                                  # T - 1 on the 8-grid, T not a multiple of 8192
W_ZERO = np.array([0.0, 0.4, 0.05, 0.0, 0.1, 0.1, 0.15, 0.1, 0.1])   # dimensions 0 and 3 weigh nothing


@pytest.fixture(autouse=True)
def forced(engine, apo):
    """loads here build the Form T copy whatever their size; the shared engine gets its default back"""
    engine.set_tuning(apo.TUNE_TWIN_T)
    yield
    engine.set_tuning(0)


def distinct(seed, n, avoid):
    """n distinct categorical evaluations Form T can index (coded dimensions from 10 levels or absent, tool_success_rate
    from 200 values), none equal to a row of `avoid`"""
    rng = np.random.default_rng(seed)
    levels = np.array([-1.0, -0.8, -0.5, -0.3, -0.2, 0.0, 0.3, 0.5, 0.8, 1.0], np.float32)
    m = n + n // 4 + 1000
    d = levels[rng.integers(0, len(levels), (m, 9))]
    d[:, 2] = rng.uniform(-1, 1, 200).astype(np.float32)[rng.integers(0, 200, m)]
    d[rng.random(d.shape) < 0.3] = np.nan
    u = d.view(np.uint32)
    seen = {r.tobytes() for r in avoid.view(np.uint32)}
    keep = []
    for i in range(m):
        k = u[i].tobytes()
        if k not in seen:
            seen.add(k)
            keep.append(i)
            if len(keep) == n:
                return d[keep]
    raise AssertionError("pool too small")


def zero_weight_rows():
    """the 120 evaluations with only dimensions 0 and 3 present: uncounted under W_ZERO"""
    levels = np.array([np.nan, -1.0, -0.8, -0.5, -0.3, -0.2, 0.0, 0.3, 0.5, 0.8, 1.0], np.float32)
    rows = []
    for a in levels:
        for b in levels:
            if np.isnan(a) and np.isnan(b):
                continue
            r = np.full(9, np.nan, np.float32)
            r[0], r[3] = a, b
            rows.append(r)
    return np.array(rows)


def tensor(seed, Cn, Tn, rare, zero_row=None):
    """[Cn][Tn] dims: rare positions (bool [Cn][Tn]) each hold a distinct evaluation seen once; row zero_row's rare ones
    are zero_weight_rows(); every other position one of NF frequent evaluations, each at least twice"""
    rng = np.random.default_rng(seed)
    zw = zero_weight_rows()
    n_zero = int(rare[zero_row].sum()) if zero_row is not None else 0
    assert n_zero <= len(zw)
    n_rare = int(rare.sum()) - n_zero
    pool = distinct(seed, NF + n_rare, zw)
    freq, other = pool[:NF], pool[NF:]
    d = np.empty((Cn, Tn, 9), np.float32)
    spots = np.flatnonzero(~rare.reshape(-1))
    assert len(spots) >= 2 * NF
    pick = rng.permutation(len(spots))
    which = np.concatenate([np.repeat(np.arange(NF), 2),
                            np.minimum(rng.geometric(1 / 300, len(spots) - 2 * NF) - 1, 1999)])   # skewed: the head
    d.reshape(-1, 9)[spots[pick]] = freq[which]
    if zero_row is not None:
        zr = np.zeros_like(rare)
        zr[zero_row] = rare[zero_row]
        d[zr] = zw[:n_zero]
        rest = rare & ~zr
    else:
        rest = rare
    d[rest] = other
    return d


def layouts(seed):
    """the main tensor: every layout of the list; about 1.4 % of the evaluations are exceptions"""
    rng = np.random.default_rng(seed)
    rare = np.zeros((C, T), bool)
    rare[0, [0, T - 1]] = True
    rare[0, rng.choice(T, 300, replace=False)] = True               # scattered
    rare[2, XBLOCK:2 * XBLOCK] = True                                # a block of exceptions
    rare[2, 100:200] = True                                          # a run longer than a warp
    rare[3, rng.choice(T, 100, replace=False)] = True               # uncounted under W_ZERO: a negative net count
    rare[4] = True                                                   # only exceptions; row 1 has none
    for c in range(5, C):
        rare[c, rng.choice(T, 50, replace=False)] = True
    return tensor(seed, C, T, rare, zero_row=3), rare


@functools.lru_cache(maxsize=1)
def main():
    return layouts(0x5EED7160)


def exact(engine, apo, Cn, call, want):
    """call()'s integers are `want` (None: not checked) and those of the TUNE_NO_TWIN_T2, TUNE_NO_TWIN_T and TUNE_NO_TWIN
    runs, with the same results"""
    engine.set_tuning(apo.TUNE_TWIN_T)
    call()
    r = call()
    p = engine.debug_partials(Cn)
    if want is not None:
        assert p == want
    try:
        for flags in (apo.TUNE_NO_TWIN_T2, apo.TUNE_NO_TWIN_T, apo.TUNE_NO_TWIN):
            engine.set_tuning(flags)
            r1 = call()
            assert engine.debug_partials(Cn) == p and same(r, r1), flags
    finally:
        engine.set_tuning(apo.TUNE_TWIN_T)
    return r


def expected_list(engine, Cn, Tn):
    """the list from resident Form T of the same tensor (apo_dims_tuples builds the same dictionary)"""
    engine.dims_tuples()
    xs, xb = [], []
    nblk = -(-Tn // XBLOCK)
    off = 0
    for c in range(Cn):
        tl, th = engine.tuples_download(c, 0, Tn)
        pos = np.flatnonzero(th)
        xs.append(np.stack([pos, tl[pos].astype(np.uint32) | (th[pos].astype(np.uint32) << 16)], 1))
        per = np.bincount(pos // XBLOCK, minlength=nblk)
        xb.append(off + np.concatenate([[0], np.cumsum(per)]))
        off += len(pos)
    return np.concatenate(xb).astype(np.uint32), np.concatenate(xs).astype(np.uint32)


def test_list_and_launches(engine, orc, apo):
    dims, rare = main()
    engine.dims_upload(dims)
    got = engine.debug_twin_t_list()
    assert got is not None
    xb, xs = got
    assert len(xs) == rare.sum()                                    # the exceptions are exactly the rare evaluations
    want_xb, want_xs = expected_list(engine, C, T)
    assert np.array_equal(xb, want_xb) and np.array_equal(xs, want_xs)
    nblk = -(-T // XBLOCK)
    row = xb.reshape(C, nblk + 1)
    assert row[1, 0] == row[1, nblk] and row[4, nblk] - row[4, 0] == T and row[2, 2] - row[2, 1] == XBLOCK
    r0 = xs[row[0, 0]:row[0, nblk]]
    assert r0[0, 0] == 0 and r0[-1, 0] == T - 1
    recs = orc.gen_records(0x5EED7161, orc.STREAM_CORPUS, 0, 1, 0, 20_000, 300, 8).reshape(-1)
    engine.corpus_upload(recs)
    r = exact(engine, apo, C, lambda: engine.score(C, 2, corpus=True), orc.score_dims_fx(dims))
    assert r.timing.launches == 2 and r.report.bad == orc.report(recs).bad


def test_windows(engine, orc, apo):
    dims, _ = main()
    engine.dims_upload(dims)
    # (4004, 100): off the 8-grid, read by K1 from the fp32 tensor
    for first, count in ((0, 1), (8, XBLOCK - 8), (XBLOCK, XBLOCK), (XBLOCK + 8, 9000), (4096, 12_288), (16_376, 0), (T - 1, 0),
                         (96, 120), (4004, 100)):
        end = first + count if count else T
        exact(engine, apo, C, lambda: engine.score(C, 1, first=first, count=count), orc.score_dims_fx(dims[:, first:end]))


def test_options(engine, orc, apo):
    dims, _ = main()
    engine.dims_upload(dims)
    exp = orc.score_dims_fx(dims)
    for recip in (True, False):
        exact(engine, apo, C, lambda: engine.score(C, 3, recip=recip), kf.fx_model(dims, recip=True) if recip else exp)
    exact(engine, apo, C, lambda: engine.score(C, 2, candidates=True), exp)
    for K in range(1, C + 1):                                       # every beam width, against K1 on the same engine
        engine.set_tuning(apo.TUNE_TWIN_T)
        r = engine.score(C, K)
        engine.set_tuning(apo.TUNE_NO_TWIN)
        assert same(r, engine.score(C, K)), K
    engine.set_tuning(apo.TUNE_TWIN_T)


def test_sessions_mix_routes(engine, orc, apo):
    dims, _ = main()
    engine.dims_upload(dims)
    sums, counts = orc.score_dims_fx(dims)

    def session(cand=False):
        engine.score_begin(C + 2)
        engine.score_accumulate(2, count=XBLOCK + 8, candidates=cand)                  # K1t2
        engine.set_tuning(apo.TUNE_NO_TWIN_T2)
        engine.score_accumulate(2, first=XBLOCK + 8, count=4000, candidates=cand)      # K1t
        engine.set_tuning(apo.TUNE_TWIN_T)
        engine.score_accumulate(2, first=XBLOCK + 4008, count=5004, candidates=cand)   # K1t2; the next start is off the grid
        engine.score_accumulate(2, first=XBLOCK + 9012, candidates=cand)               # K1
        return engine.score_finish(C + 2, 3, corpus=True, candidates=cand)

    want = ([0, 0] + list(sums), [0, 0] + list(counts))
    exact(engine, apo, C + 2, session, want)
    exact(engine, apo, C + 2, lambda: session(True), want)


def test_weights_set_after_the_load(engine, orc, apo):
    """under W_ZERO row 3's exceptions are uncounted and their low-plane aliases counted: the count correction is negative"""
    dims, _ = main()
    engine.dims_upload(dims)
    try:
        for w in (W_ZERO, orc.weights()):
            engine.set_weights(w)
            want = orc.score_dims_fx(dims, w=w)
            exact(engine, apo, C, lambda: engine.score(C, C), want)
            exact(engine, apo, C, lambda: engine.score(C, C, recip=True), kf.fx_model(dims, w=w, recip=True))
        engine.set_weights(W_ZERO)
        engine.score(C, 1)
        assert engine.debug_partials(C)[1][3] <= T - 100              # row 3 lost the counts of its uncounted exceptions
    finally:
        engine.set_weights(orc.weights())


def test_eligibility_bound(engine, orc, apo):
    """at most 1/64 of the evaluations as exceptions: the list; one more: K1t from both planes, the same results"""
    Cb = 64
    for extra in (0, 1):
        rare = np.zeros((Cb, T), bool)
        rare[4] = True                                               # T = Cb * T / 64 exceptions
        if extra:
            rare[0, 5] = True
        dims = tensor(0x5EED7162, Cb, T, rare)
        engine.dims_upload(dims)
        got = engine.debug_twin_t_list()
        assert (got is None) == bool(extra)
        if got is not None:
            assert len(got[1]) * 64 == Cb * T
        exact(engine, apo, Cb, lambda: engine.score(Cb, 2), orc.score_dims_fx(dims))


def test_small_dictionary_takes_the_2_byte_route(engine, orc, apo):
    """<= 2^16 distinct evaluations: an empty list (none held), and K1t2 reads the copy without a correction"""
    dims = orc.gen_dims(0x5EED7163, 0, 4, 0, 30_000, 300, 8)
    engine.dims_upload(dims)
    assert engine.debug_twin_t_list() is None
    exact(engine, apo, 4, lambda: engine.score(4, 2), orc.score_dims_fx(dims))


def test_every_drop_path_releases_the_list(engine, orc, apo):
    import torch
    dims, _ = main()
    engine.dims_upload(dims)
    assert engine.debug_twin_t_list() is not None
    engine.dims_compact()
    assert engine.debug_twin_t_list() is None
    engine.dims_upload(dims)
    assert engine.debug_twin_t_list() is not None
    pitch = (T + 3) // 4 * 4
    buf = torch.zeros((C, pitch, 9), dtype=torch.float32, device="cuda")
    buf[:, :T] = torch.from_numpy(dims).cuda()
    engine.dims_attach(buf.data_ptr(), C, T, pitch)
    assert engine.debug_twin_t_list() is None
    del buf
    engine.dims_upload(dims)
    assert engine.debug_twin_t_list() is not None
    engine.set_tuning(apo.TUNE_TWIN_T | apo.TUNE_NO_TWIN_T2)         # a load with the flag builds none
    engine.dims_upload(dims)
    assert engine.debug_twin_t_list() is None
    engine.dims_upload(dims)
    engine.set_tuning(apo.TUNE_TWIN_T | apo.TUNE_NO_TWIN_T)           # a load without the Form T copy holds no list
    engine.dims_upload(dims)
    assert engine.debug_twin_t_list() is None
    engine.set_tuning(apo.TUNE_TWIN_T)
    engine.dims_upload(orc.gen_dims(0x5EED7164, 0, 3, 0, 10_000, 300, 8))   # a later load replaces it
    assert engine.debug_twin_t_list() is None


GRID_SCRIPT = r"""
import hashlib, importlib, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {here!r})
import test_gpu_twin_t_list as t
apo = importlib.import_module("senweaver-ide_b200")
e = apo.Engine(0)
e.set_tuning(apo.TUNE_TWIN_T)
dims, _ = t.layouts(0x5EED7160)
e.dims_upload(dims)
xb, xs = e.debug_twin_t_list()
h = hashlib.sha256(xb.tobytes() + xs.tobytes())
for first, count in ((0, 0), (4096, 20_000 - 4096)):
    e.score(t.C, 3, first=first, count=count)
    h.update(repr(e.debug_partials(t.C)).encode())
e.close()
print(h.hexdigest())
"""


def test_grid_independence(apo):
    """the list's bytes and the scores for forced grids of 1 and 7 CTAs (APO_K1_GRID, read once per process)"""
    script = GRID_SCRIPT.format(root=ROOT, here=HERE)
    out = []
    for grid in (None, "1", "7"):
        env = dict(os.environ)
        env.pop("APO_K1_GRID", None)
        if grid:
            env["APO_K1_GRID"] = grid
        r = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, env=env, cwd=ROOT, timeout=900)
        assert r.returncode == 0, r.stderr[-2000:]
        out.append(r.stdout.split()[-1])
    assert out[0] == out[1] == out[2]
