"""K1t2's slot layout at its edges (-m gpu, csrc/apo_kernels.h).  The tensor holds 65 536 frequent evaluations (every rank
below 2^16 occurs, so the entries h - 1 / h, the one in the last shared-memory slot and the one after it, end - 1 / end and
2^16 - 1 all do), rare ones seen once (the exceptions), and one row made only of evaluations whose entry has no slot (the
second list).  Every result must equal the oracle's integers (the numpy model for recip) and those of K1t, K1q and K1 on the
same engine: windows on the 8-grid off the 128- and 256-grids, ragged row ends, recip, weights set after the load, every K,
and forced CTA cuts (APO_K1_GRID)."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

import k1_fixtures as kf
import slot_model as sm
import test_gpu_twin_t_list as tl
from test_gpu_dims_twin import same

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
C, T = 96, 20_011                                   # ragged: T - 3 on the 8-grid
TAIL_ROW = 5
H = sm.SLOT_H
END = sm.slot_end(1 << 20, H)
LAST_SHARED = sm.HOT_MAX - 1 - (sm.REP - 1) * H - 1   # the entry in the last shared-memory slot


@pytest.fixture(autouse=True)
def forced(engine, apo):
    engine.set_tuning(apo.TUNE_TWIN_T)
    yield
    engine.set_tuning(0)


def ranks(engine, Cn, Tn):
    """the dictionary index of every evaluation (resident Form T of the same tensor builds the same dictionary)"""
    engine.dims_tuples()
    out = np.empty((Cn, Tn), np.int64)
    for c in range(Cn):
        lo, hi = engine.tuples_download(c, 0, Tn)
        out[c] = lo.astype(np.int64) | (hi.astype(np.int64) << 16)
    return out


@functools.lru_cache(maxsize=1)
def build():
    """[C][T] dims: END head evaluations seen at least 4 times, the 2^16 - END
    after them 3 times each (ranks END .. 2^16 - 1: no slot), filling row TAIL_ROW and a few places elsewhere, and rare ones
    seen once (the exceptions)"""
    rng = np.random.default_rng(0x5EED7170)
    n_tail = 65536 - END
    rare = np.zeros((C, T), bool)
    rare[0, [0, T - 1]] = True
    for c in range(1, C):
        if c != TAIL_ROW:
            rare[c, rng.choice(T, 40, replace=False)] = True
    pool = tl.distinct(0x5EED7170, 65536 + int(rare.sum()), tl.zero_weight_rows())
    head, tail, other = pool[:END], pool[END:65536], pool[65536:]
    tail_evals = rng.permutation(np.repeat(np.arange(n_tail), 3))
    dims = np.empty((C, T, 9), np.float32)
    dims[TAIL_ROW] = tail[tail_evals[:T]]
    spots = np.flatnonzero(~rare.reshape(-1) & (np.arange(C * T) // T != TAIL_ROW))
    spots = spots[rng.permutation(len(spots))]
    left = tail_evals[T:]
    dims.reshape(-1, 9)[spots[:len(left)]] = tail[left]
    spots = spots[len(left):]
    which = np.concatenate([np.repeat(np.arange(END), 4),
                            np.minimum(rng.geometric(1 / 300, len(spots) - 4 * END) - 1, END - 1)])
    dims.reshape(-1, 9)[spots] = head[which]
    dims[rare] = other
    return dims


def test_layout_edges_are_present(engine):
    dims = build()
    engine.dims_upload(dims)
    idx = ranks(engine, C, T)
    assert np.all((idx[TAIL_ROW] >= END) & (idx[TAIL_ROW] < 65536))
    counts = np.bincount(idx.reshape(-1))
    h, end = sm.choose_h(counts, C * T)
    assert (h, end) == (H, END)
    for e in (H - 1, H, LAST_SHARED, LAST_SHARED + 1, END - 1, END, 65535, 65536):
        assert counts[e] > 0, e


def test_calls_against_oracle(engine, orc, apo):
    dims = build()
    engine.dims_upload(dims)
    assert engine.debug_twin_t_list() is not None
    tl.exact(engine, apo, C, lambda: engine.score(C, 2), orc.score_dims_fx(dims))
    for first, count in ((8, 0), (136, 5000), (264, 16_384), (4008, T - 4008), (16_384, 3), (T - 3, 0)):
        end = first + count if count else T
        tl.exact(engine, apo, C, lambda: engine.score(C, 1, first=first, count=count), orc.score_dims_fx(dims[:, first:end]))
    for recip in (True, False):
        tl.exact(engine, apo, C, lambda: engine.score(C, 3, recip=recip), kf.fx_model(dims, recip=True) if recip else orc.score_dims_fx(dims))
    for K in (1, 7, C):
        engine.set_tuning(apo.TUNE_TWIN_T)
        r = engine.score(C, K)
        engine.set_tuning(apo.TUNE_NO_TWIN)
        assert same(r, engine.score(C, K)), K
    engine.set_tuning(apo.TUNE_TWIN_T)


def test_weights_set_after_the_load(engine, orc, apo):
    dims = build()
    engine.dims_upload(dims)
    try:
        for w in (tl.W_ZERO, orc.weights()):
            engine.set_weights(w)
            tl.exact(engine, apo, C, lambda: engine.score(C, C), orc.score_dims_fx(dims, w=w))
            tl.exact(engine, apo, C, lambda: engine.score(C, 2, recip=True), kf.fx_model(dims, w=w, recip=True))
    finally:
        engine.set_weights(orc.weights())


GRID_SCRIPT = r"""
import importlib, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {here!r})
import test_gpu_slot_layout as t
apo = importlib.import_module("senweaver-ide_b200")
e = apo.Engine(0)
e.set_tuning(apo.TUNE_TWIN_T)
dims = t.build()
e.dims_upload(dims)
out = []
for first, count in ((0, 0), (136, 12_000), (8, 0)):
    e.score(t.C, 3, first=first, count=count)
    out.append(e.debug_partials(t.C))
e.set_tuning(apo.TUNE_TWIN_T | apo.TUNE_NO_TWIN)
for first, count in ((0, 0), (136, 12_000), (8, 0)):
    e.score(t.C, 3, first=first, count=count)
    out.append(e.debug_partials(t.C))
e.close()
print("same" if out[:3] == out[3:] else "differ")
"""


def test_grid_cuts():
    """forced grids of 1, 5 and 97 CTAs (APO_K1_GRID, read once per process): K1t2 against K1 in the same process"""
    for grid in ("1", "5", "97"):
        env = dict(os.environ, APO_K1_GRID=grid)
        r = subprocess.run([sys.executable, "-c", GRID_SCRIPT.format(root=ROOT, here=HERE)], env=env, capture_output=True,
                           text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        assert r.stdout.strip().splitlines()[-1] == "same", (grid, r.stdout[-500:])
