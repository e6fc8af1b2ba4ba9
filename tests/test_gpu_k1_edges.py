"""K1 (Form D), K1r (Form R / R16), K1q (Form Q) and the K3 tail at their edges on the H100 (-m gpu), on the hand-built tensors
of tests/k1_fixtures.py.

Every case compares debug_partials (exact sums and counts) with the oracle's integers, the scores bit for bit with
sharding.scores_from_partials of those integers and the top-K with sharding.topk_indices -- no tolerance.  APO_SCORE_RECIP
is compared with the numpy restatement of the Form D arithmetic (k1_fixtures.fx_model) for Form D / Q, and with variant 0
for Form R / R16.

- every variant of K1 (D / R / R16) and K1q, with and without recip: resident windows of T = TILE - 8 ... 2 TILE + 1 starting
  off the tile grid, short rows of 300 candidates, one session of two windows and one host-streamed call;
- the same kernels with the grid forced down to 1, 2, 3 and 7 CTAs (APO_K1_GRID, read once per process: a subprocess each),
  so that CTA ranges start and end inside candidates and the stage ring wraps its phase many times;
- sums past 2^64, 2^72 and 2^83, exact binary64 ties with and without a sticky bit in both branches of limbs_to_double;
- K3 at C = 1 ... 4096 and on both sides of the 64 KB result block, K = 0, 1, a K inside a tie group and C, through every
  kernel that finalises: the fused tail of the scoring launch (with and without a corpus), k_detect6_tiles and the
  grid-stride k_detect6 (sessions with corpora of 9000 and 500 records) and k_finalize (a session without corpus, and
  TUNE_NO_FUSE);
- out-of-domain Form D / Q evaluations (finalReward of 512 or more, below -512, +-inf) fail the call with APO_E_ARG and leave the
  handle exact."""
import importlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import k1_fixtures as kf

pytestmark = pytest.mark.gpu

sharding = importlib.import_module("senweaver-ide_b200.sharding")
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
APO_E_ARG = -1
FORMS = [("D", v) for v in kf.TILES_K1] + [("R", v) for v in kf.TILES_K1] + [("R16", v) for v in kf.TILES_K1] + \
        [("Q", v) for v in kf.TILES_KQ]


def tile_of(form, variant):
    return (kf.TILES_KQ if form == "Q" else kf.TILES_K1)[variant]


def check(engine, res, want, C, K=None):
    sums, counts = want
    assert engine.debug_partials(C) == (sums, counts)
    scores = sharding.scores_from_partials(sums, counts)
    assert res.scores.tobytes() == scores.tobytes()
    assert [int(x) for x in res.counts] == counts
    K = len(res.topk) if K is None else K
    assert np.array_equal(res.topk[:K], sharding.topk_indices(scores, K))


def refused(apo, call):
    with pytest.raises(apo.ApoError) as ei:
        call()
    assert ei.value.code == APO_E_ARG


class Data:
    """one tensor in the layout a form is scored from, and its reference"""

    def __init__(self, apo, form, C, T, seed=0):
        self.form, self.apo = form, apo
        if form in ("R", "R16"):
            self.recs = kf.shape_records(C, T, seed)
            self.rows = apo.pack16(self.recs) if form == "R16" else self.recs
            self.ref_recs = kf.oracle.unpack16(self.rows) if form == "R16" else self.recs
        else:
            self.dims = kf.shape_dims(C, T, seed) if T > 8 else kf.short_dims(C, T, seed)

    @classmethod
    def of_dims(cls, apo, form, dims):
        d = cls.__new__(cls)
        d.form, d.apo, d.dims = form, apo, np.ascontiguousarray(dims, np.float32)
        return d

    def upload(self, engine):
        if self.form == "D":
            engine.dims_upload(self.dims)
        elif self.form == "Q":
            engine.dims_upload_compact(self.dims)
            assert engine.dims_layout() == 2
        elif self.form == "R":
            engine.rollouts_upload(self.rows)
        else:
            engine.rollouts16_upload(self.rows)

    @property
    def source(self):
        return self.apo.SRC_ROLLOUTS if self.form in ("R", "R16") else self.apo.SRC_DIMS

    def want(self, a=0, n=None, recip=False):
        if self.form in ("R", "R16"):
            r = self.ref_recs[:, a:None if n is None else a + n]
            return kf.oracle.score_records_fx(np.ascontiguousarray(r))
        d = self.dims[:, a:None if n is None else a + n]
        return kf.fx_model(d, recip=True) if recip else kf.oracle_fx(d)

    def stream(self, engine, K, variant, recip):
        if self.form == "D":
            return engine.score_host(np.ascontiguousarray(self.dims), K, variant=variant, recip=recip)
        if self.form == "Q":
            q8, d2, li, book = self.apo.compact_encode_host(self.dims)
            return engine.score_host_compact(q8, d2, li, book, K, recip=recip)
        return engine.score_host_records(np.ascontiguousarray(self.rows), K, variant=variant, recip=recip)


def score_variant(engine, data, C, K, variant, recip, first=0, count=0):
    return engine.score(C, K, source=data.source, variant=variant, recip=recip, first=first, count=count)


def want_for(engine, data, C, variant, recip, first=0, count=None):
    """the reference of a window: the oracle (or the numpy model for Form D / Q recip); Form R / R16 recip: variant 0"""
    if recip and data.form in ("R", "R16"):
        score_variant(engine, data, C, 1, 0, True, first, count or 0)
        got = engine.debug_partials(C)
        ref = data.want(first, count)
        assert got[1] == ref[1]
        assert all(abs(a - b) <= 2 ** 11 * sum(ref[1]) for a, b in zip(got[0], ref[0]))
        return got
    return data.want(first, count, recip)


@pytest.mark.parametrize("recip", [False, True])
@pytest.mark.parametrize("form,variant", FORMS)
def test_every_variant_at_tile_edges(engine, apo, form, variant, recip):
    tile = tile_of(form, variant)
    align = 8 if form == "Q" else 4
    C = 4
    starts = kf.window_starts(tile, align)
    data = Data(apo, form, C, max(starts) + 2 * tile + 16, seed=variant)
    data.upload(engine)
    for k, T in enumerate(kf.t_edges(tile)):
        first = starts[k % len(starts)]
        r = score_variant(engine, data, C, 2, variant, recip, first, T)
        check(engine, r, want_for(engine, data, C, variant, recip, first, T), C)
    # a session of two windows cut off the tile grid, then one host-streamed call of a whole tensor
    cut = tile + 3 * align
    want = want_for(engine, data, C, variant, recip, 0, 2 * tile + 1)
    engine.score_begin(C)
    engine.score_accumulate(0, source=data.source, recip=recip, variant=variant, first=cut, count=2 * tile + 1 - cut)
    engine.score_accumulate(0, source=data.source, recip=recip, variant=variant, first=0, count=cut)
    check(engine, engine.score_finish(C, 2), want, C)
    part = Data.__new__(Data)
    part.__dict__.update(data.__dict__)
    if form in ("R", "R16"):
        part.rows = np.ascontiguousarray(data.rows[:, :tile + 1])
        part.ref_recs = np.ascontiguousarray(data.ref_recs[:, :tile + 1])
    else:
        part.dims = np.ascontiguousarray(data.dims[:, :tile + 1])
    if form == "Q" or not recip or form == "D":
        check(engine, part.stream(engine, 2, variant, recip), part.want(recip=recip), C)
    # short rows: one tile per candidate, every CTA's range crosses many candidates
    for T in (1, 3, 7):
        short = Data(apo, form, 300, T, seed=T)
        short.upload(engine)
        r = score_variant(engine, short, 300, 4, variant, recip)
        check(engine, r, want_for(engine, short, 300, variant, recip), 300)


GRID_SCRIPT = r"""
import importlib, json, sys
sys.path[:0] = [sys.argv[1], sys.argv[2]]
import numpy as np
import k1_fixtures as kf
from test_gpu_k1_edges import Data, FORMS, tile_of
apo = importlib.import_module("senweaver-ide_b200")
e = apo.Engine(0)
out = {}
for form, v in FORMS:
    tile = tile_of(form, v)
    for C, T in ((3, 2 * tile + 1), (2, 5 * tile - 8), (300, 7)):
        d = Data(apo, form, C, T, seed=v)
        d.upload(e)
        e.score(C, 1, source=d.source, variant=v)
        s, n = e.debug_partials(C)
        out[f"{form}/{v}/{C}/{T}"] = [[str(x) for x in s], n]
e.close()
print(json.dumps(out))
"""


@pytest.mark.parametrize("grid", [1, 2, 3, 7])
def test_forced_grid(apo, orc, grid):
    """APO_K1_GRID (read once per process) forces K1 / K1r / K1q down to `grid` CTAs: every variant, full and partial
    tiles, and 300 short candidates per CTA range; the integers are the oracle's"""
    env = dict(os.environ, APO_K1_GRID=str(grid))
    p = subprocess.run([sys.executable, "-c", GRID_SCRIPT, ROOT, HERE], env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-3000:]
    got = json.loads(p.stdout.strip().splitlines()[-1])
    for form, v in FORMS:
        tile = tile_of(form, v)
        for C, T in ((3, 2 * tile + 1), (2, 5 * tile - 8), (300, 7)):
            s, n = got[f"{form}/{v}/{C}/{T}"]
            assert ([int(x) for x in s], n) == Data(apo, form, C, T, seed=v).want(), (form, v, C, T)


@pytest.mark.parametrize("form,variant", [("D", v) for v in kf.TILES_K1] + [("Q", 0), ("Q", 3), ("Q", 4)])
def test_extreme_sums_and_binary64_ties(engine, apo, form, variant):
    for dims in (kf.extreme_dims(), kf.tie_dims()):
        data = Data.of_dims(apo, form, dims)
        C = dims.shape[0]
        data.upload(engine)
        for recip in (False, True):
            r = score_variant(engine, data, C, C, variant, recip)
            check(engine, r, data.want(recip=recip), C)
        if variant == 0:
            check(engine, data.stream(engine, C, 0, False), data.want(), C)
            engine.score_begin(C)
            engine.score_accumulate(0, first=1024)
            engine.score_accumulate(0, first=0, count=1024)
            check(engine, engine.score_finish(C, C), data.want(), C)


def test_sums_past_2_83(engine, apo):
    data = Data.of_dims(apo, "D", kf.huge_dims())
    want, want_r = data.want(), data.want(recip=True)
    assert want[0][0] > 1 << 83
    data.upload(engine)
    for v in kf.TILES_K1:
        check(engine, score_variant(engine, data, 2, 2, v, False), want, 2)
    check(engine, score_variant(engine, data, 2, 2, 0, True), want_r, 2)
    check(engine, data.stream(engine, 2, 0, False), want, 2)
    q = Data.of_dims(apo, "Q", data.dims)
    q.upload(engine)
    check(engine, score_variant(engine, q, 2, 2, 0, False), want, 2)


# ------------------------------------------------------------------------------------------------ K3
def corpus(orc, n):
    return orc.gen_records(0x5EED2000 + n, orc.STREAM_CORPUS, 0, 1, 0, n, 300, 8).reshape(-1)


def finalise(engine, apo, orc, path, C, K):
    if path == "fused":
        return engine.score(C, K)
    if path == "fused_corpus":
        engine.corpus_upload(corpus(orc, 500))
        r = engine.score(C, K, corpus=True)
        assert r.timing.launches == 1
        return r
    if path == "no_fuse":
        try:
            engine.set_tuning(apo.TUNE_NO_FUSE)
            r = engine.score(C, K)
            assert r.timing.launches == 2
            return r
        finally:
            engine.set_tuning(0)
    n = {"tiles": 9000, "gridstride": 500, "finalize": 0}[path]
    if n:
        engine.corpus_upload(corpus(orc, n))
    engine.score_begin(C)
    engine.score_accumulate(0)
    return engine.score_finish(C, K, corpus=n > 0)


@pytest.mark.parametrize("path", ["fused", "fused_corpus", "tiles", "gridstride", "finalize", "no_fuse"])
def test_k3_sizes_ties_and_topk(engine, apo, orc, path):
    for C in kf.k3_sizes():
        for mode in (("mixed", "sparse", "equal") if C in (1025, 2049, 4096) else ("mixed",)):
            dims = kf.key_dims(C, mode)
            want = kf.oracle_fx(dims)
            assert want == kf.key_targets(C, mode)
            scores = sharding.scores_from_partials(*want)
            engine.dims_upload(dims)
            for K in kf.k_values(scores):
                r = finalise(engine, apo, orc, path, C, K)
                check(engine, r, want, C, K)


# ------------------------------------------------------------------------------------------------ domain
BAD = {"p512": np.float32(512.0), "n512": np.nextafter(np.float32(-512.0), np.float32(-np.inf)), "pinf": np.float32(np.inf), "ninf": np.float32(-np.inf)}


@pytest.mark.parametrize("dim", [0, 2])
@pytest.mark.parametrize("where", ["full_tile", "ragged_tail"])
@pytest.mark.parametrize("value", list(BAD))
@pytest.mark.parametrize("form", ["D", "Q"])
def test_out_of_domain_evaluations_are_refused(engine, apo, form, value, where, dim):
    """a finalReward of 512 or more, below -512 or +-inf would overflow the int64 pre-add or saturate rint(fr * 2^52): APO_E_ARG on the
    resident call, a session and the host-streamed call; the same tensor without it is exact afterwards"""
    tile = tile_of(form, 0)
    C, T = 3, 2 * tile + 5
    data = Data(apo, form, C, T)
    clean = data.dims.copy()
    data.dims[1, 100 if where == "full_tile" else T - 2] = kf.single(BAD[value], dim)
    data.upload(engine)
    refused(apo, lambda: engine.score(C, 1))
    if "inf" in value:                                   # ws * RN(1/tw) of a finite value just outside may round inside
        refused(apo, lambda: engine.score(C, 1, recip=True))
    engine.score_begin(C)
    engine.score_accumulate(0, first=0, count=tile)
    engine.score_accumulate(0, first=tile)
    refused(apo, lambda: engine.score_finish(C, 1))
    refused(apo, lambda: data.stream(engine, 1, 0, False))
    ok = Data.of_dims(apo, form, clean)
    ok.upload(engine)
    check(engine, engine.score(C, 2), ok.want(), C)
    check(engine, ok.stream(engine, 2, 0, False), ok.want(), C)
    # the largest in-domain values next to the refused ones are scored
    near = clean.copy()
    near[1, 100] = kf.single(np.float32(-512.0) if value[0] == "n" else kf.MAXF, dim)      # -512 itself is inside
    ok = Data.of_dims(apo, form, near)
    ok.upload(engine)
    check(engine, engine.score(C, 2), ok.want(), C)
