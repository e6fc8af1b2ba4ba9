"""K1h's corpus digest pass at small shares per CTA (-m gpu).

With the corpus report, each K1h CTA runs its share of the digest entries either on its last warp beside the pair stream
(four entries in flight per lane, set-up and flush by that warp alone) or, when its pairs are few for its share, on all
its warps after the stream.  Digests of 1, 2, 7, 31, 32 and 33 entries per CTA, and 127, 128 and 129 (the warp's four
entries in flight per lane), at forced grids of 1 and 7 CTAs: the dims of test_gpu_count_route have ~10 k pairs per CTA at
7 CTAs and ~70 k at 1, so both passes are reached.  Every report must be byte-equal to the corpus scan's
(TUNE_NO_CORPUS_DIGEST) and to the stand-alone k_corpus_digest's (TUNE_NO_TWIN_H), with the same scores and top-K, in
one launch, and field-equal to the oracle."""
import json
import os
import subprocess
import sys

import pytest

import flagship_fixtures as ff
from test_gpu_candidate_corpus import check_oracle

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
PER_CTA = (1, 2, 7, 31, 32, 33, 127, 128, 129)
GRIDS = (1, 7)
IDX_BASE = 11

SCRIPT = r"""
import importlib, json, sys
sys.path[:0] = [sys.argv[1], sys.argv[2]]
import flagship_fixtures as ff
import test_gpu_count_route as cr
apo = importlib.import_module("senweaver-ide_b200")
e = apo.Engine(0)
e.set_tuning(apo.TUNE_TWIN_T)
e.dims_upload(cr.build())
assert e.debug_twin_h() is not None
out = []
for nkeys in json.loads(sys.argv[3]):
    e.set_tuning(apo.TUNE_TWIN_T)
    e.corpus_upload(ff.cycled(ff.FEW_T, nkeys), int(sys.argv[4]))
    for _ in range(3):                                   # the second reported call builds the digest, the third reads it
        r = e.score(cr.C, 2, corpus=True)
    dig = e.debug_corpus_digest()
    row = {"entries": 0 if dig is None else len(dig[0]), "launches": int(r.timing.launches)}
    e.set_tuning(apo.TUNE_TWIN_T | apo.TUNE_NO_CORPUS_DIGEST)
    scan = e.score(cr.C, 2, corpus=True)
    e.set_tuning(apo.TUNE_TWIN_T | apo.TUNE_NO_TWIN_H)
    alone = e.score(cr.C, 2, corpus=True)
    for name, x in (("k1h", r), ("scan", scan), ("alone", alone)):
        row[name] = {"report": bytes(x.report).hex(), "scores": x.scores.tobytes().hex(), "topk": x.topk.tolist()}
    out.append(row)
e.close()
print(json.dumps(out))
"""


@pytest.mark.parametrize("grid", GRIDS)
def test_digest_shares(apo, orc, grid):
    nkeys = [k * grid for k in PER_CTA]
    p = subprocess.run([sys.executable, "-c", SCRIPT, ROOT, HERE, json.dumps(nkeys), str(IDX_BASE)],
                       env=dict(os.environ, APO_K1_GRID=str(grid)), capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-3000:]
    out = json.loads(p.stdout.strip().splitlines()[-1])
    for n, row in zip(nkeys, out):
        assert row["entries"] == n and row["launches"] == 1, (grid, n, row["entries"], row["launches"])
        assert row["k1h"] == row["scan"] == row["alone"], (grid, n)
        ref = orc.report(ff.cycled(ff.FEW_T, n), idx_base=IDX_BASE, nthreads=16)
        check_oracle(apo, apo.engine.CorpusReport.from_buffer_copy(bytes.fromhex(row["k1h"]["report"])), ref)
