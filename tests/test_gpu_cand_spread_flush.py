"""The per-candidate reward spread's run-limit flush (csrc/apo_cand.cu k_cand_spread): one CTA over 600 M evaluations of
constant rows at fr = -512 and 512 - 2^-15, so that every warp flushes mid-row after 65 536 tiles with lane sums past 2^143.

The rows are a 21.6 GB Form D tensor on the device, attached to a fresh engine in a process of its own (APO_K1_GRID is read
once per process).  That needs the device nearly to itself, so this check sits in its own module, which runs before the
modules whose tests leave large tensors on the session's shared engine."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))

FLUSH_SCRIPT = r"""
import json, sys
sys.path[:0] = [sys.argv[1], sys.argv[2]]
from importlib import import_module
import torch
import spread_fixtures as sf
apo = import_module("senweaver-ide_b200")
T = 300_000_000
buf = torch.full((2, T, 9), float("nan"), dtype=torch.float32, device="cuda:0")
buf[0, :, 1] = -512.0
buf[1, :, 1] = sf.F32_BELOW_512
torch.cuda.synchronize()
e = apo.Engine(0)
try:
    e.set_weights(sf.w_one())
    e.dims_attach(buf.data_ptr(), 2, T, T)
    r = e.score(2, 1, spread=True)
    got = [[int(s.n), s.sum, s.sum_sq, s.variance.hex(), s.stdDev.hex(), s.stdErr.hex(), s.mean.hex()] for s in r.spread]
finally:
    e.close()
want = [sf.constant_model(T, v) for v in (-512.0, sf.F32_BELOW_512)]
want = [[m["n"], m["S1"], m["S2"], m["variance"].hex(), m["stdDev"].hex(), m["stdErr"].hex(), m["mean"].hex()] for m in want]
print(json.dumps({"ok": got == want, "got": str(got), "want": str(want)}))
"""


def test_run_flush_at_one_cta_over_600M_evaluations():
    """one CTA of 8 warps over C = 2 constant rows of T = 3e8 at -512 and 512 - 2^-15 (K1 on an attached tensor): ~73 000
    tiles per warp, so every warp flushes mid-row after 65 536 tiles; per-lane sums pass 2^143 inside a run, the candidate's
    S2 ~ 2^150, M = 0 exactly"""
    env = dict(os.environ, APO_K1_GRID="1")
    p = subprocess.run([sys.executable, "-c", FLUSH_SCRIPT, ROOT, HERE], env=env, capture_output=True, text=True, timeout=3000)
    assert p.returncode == 0, p.stderr[-4000:]
    out = json.loads(p.stdout.strip().splitlines()[-1])
    assert out["ok"], out
