"""K1q's table addressing on the Form W copy (-m gpu).  Each evaluation turns its word into six product-table addresses (one
PRMT per nibble), a swizzled prefix-table slot and a LUT entry found by a multiply-gather of the eight presence flags.  These
cases put every code, every presence mask and both division paths through that addressing, on full tiles and a short last
tile, and check the integers against the oracle (the numpy model for recip) and against the TUNE_NO_TWIN run of the same
engine (K1 on the fp32 tensor); a profiler record shows that the Form W instantiation ran."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import k1_fixtures as kf
from test_gpu_dims_word import NAN, TILE, exact

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CODED = (0, 1, 3, 4, 5, 6, 7, 8)                      # dimension of nibble k
POW2 = 2.0 ** np.arange(9)                            # the total weight of a mask is the mask: 511 distinct LUT entries
ALL_ONES = np.array([0.3, 0.1, 0.05, 0.05, 0.1, 0.1, 0.1, 0.1, 0.1])   # full mask: total 0.9999999999999999, flagged negative


def code_dims(T=2 * TILE + 37, seed=5):
    """[8][T][9]: candidate k walks nibble k through its 15 values and absence (t % 16), one dimension varied at a time; the
    other coded dimensions hold one of those values, tool_success_rate a few ratios and absence"""
    rng = np.random.default_rng(seed)
    vals = np.linspace(-1.0, 1.0, 15).astype(np.float32)
    d = np.empty((8, T, 9), np.float32)
    t = np.arange(T)
    for k, dim in enumerate(CODED):
        d[k, :, :] = vals[(3 * np.arange(9) + k) % 15]
        d[k, :, dim] = np.where(t % 16 == 15, NAN, vals[np.minimum(t % 16, 14)])
        d[k, :, 2] = np.array([0.0, 0.5, -1.0 / 3, NAN], np.float32)[rng.integers(0, 4, T)]
    for dim in CODED:                                  # every value of every coded dimension occurs: codes 0-14 are all used
        assert len(np.unique(d[:, :, dim][~np.isnan(d[:, :, dim])])) == 15
    return d


def mask_dims(T=3 * TILE + 101, C=3, seed=9):
    """[C][T][9]: every presence mask of the nine dimensions in a shuffled order per candidate, a few values per dimension"""
    rng = np.random.default_rng(seed)
    levels = np.array([0.25, -0.5, 1.0, -1.0, 0.0], np.float32)
    d = np.empty((C, T, 9), np.float32)
    for c in range(C):
        m = np.concatenate([rng.permutation(512) for _ in range(T // 512 + 1)])[:T]
        d[c] = levels[rng.integers(0, 5, (T, 9))]
        d[c, :, 2] = np.array([0.0, 0.75, -0.125], np.float32)[rng.integers(0, 3, T)]
        for i in range(9):
            d[c, (m >> i) & 1 == 0, i] = NAN
    return d


def want(orc, dims, w, recip):
    return kf.fx_model(dims, w=w, recip=True) if recip else orc.score_dims_fx(dims, w=w)


@pytest.fixture
def weights(engine, orc):
    yield lambda w: engine.set_weights(w)
    engine.set_weights(orc.weights())


@pytest.mark.parametrize("recip", [False, True])
def test_every_code_in_every_nibble(engine, orc, apo, weights, recip):
    dims = code_dims()
    engine.dims_upload(dims)
    assert engine.dims_layout() == 1
    for w in (None, POW2):
        weights(orc.weights() if w is None else w)
        exact(engine, apo, 8, lambda: engine.score(8, 8, recip=recip), want(orc, dims, w, recip))


@pytest.mark.parametrize("recip", [False, True])
def test_every_mask_has_its_own_lut_entry(engine, orc, apo, weights, recip):
    dims = mask_dims()
    engine.dims_upload(dims)
    assert engine.dims_layout() == 1
    weights(POW2)
    exact(engine, apo, 3, lambda: engine.score(3, 3, recip=recip), want(orc, dims, POW2, recip))
    for first, count in ((0, TILE), (TILE - 8, TILE + 5)):      # one full tile; a window whose last tile is short
        part = dims[:, first:first + count]
        exact(engine, apo, 3, lambda: engine.score(3, 1, recip=recip, first=first, count=count), want(orc, part, POW2, recip))


@pytest.mark.parametrize("recip", [False, True])
def test_negative_reciprocal_masks(engine, orc, apo, weights, recip):
    """the full mask's reciprocal is flagged negative: without recip its groups of four take the generic division"""
    dims = mask_dims(seed=10)
    engine.dims_upload(dims)
    weights(ALL_ONES)
    exact(engine, apo, 3, lambda: engine.score(3, 3, recip=recip), want(orc, dims, ALL_ONES, recip))


GRID_SCRIPT = r"""
import importlib, json, sys
sys.path[:0] = [sys.argv[1], sys.argv[2]]
import numpy as np
import test_gpu_dims_word_lookup as t
apo = importlib.import_module("senweaver-ide_b200")
e = apo.Engine(0)
out = {}
for name, dims, w in (("codes", t.code_dims(), None), ("masks", t.mask_dims(), t.POW2)):
    e.dims_upload(dims)
    assert e.dims_layout() == 1
    if w is not None:
        e.set_weights(w)
    for recip in (0, 1):
        e.score(dims.shape[0], 1, recip=bool(recip))
        s, n = e.debug_partials(dims.shape[0])
        out[f"{name}/{recip}"] = [[str(x) for x in s], n]
e.close()
print(json.dumps(out))
"""


@pytest.mark.parametrize("grid", [1, 7])
def test_forced_grid(orc, grid):
    """APO_K1_GRID (read once per process) forces K1q on the word copy down to `grid` CTAs"""
    env = dict(os.environ, APO_K1_GRID=str(grid))
    p = subprocess.run([sys.executable, "-c", GRID_SCRIPT, ROOT, HERE], env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-3000:]
    got = json.loads(p.stdout.strip().splitlines()[-1])
    for name, dims, w in (("codes", code_dims(), None), ("masks", mask_dims(), POW2)):
        for recip in (0, 1):
            s, n = got[f"{name}/{recip}"]
            assert ([int(x) for x in s], n) == tuple(want(orc, dims, w, bool(recip))), (name, recip)
