"""The run-limit flush of the paired comparison per record group (csrc/apo_cand.cu k_cand_group_pairs): one CTA over 600 M
evaluations of constant rows at fr = 512 - 2^-15 and -512 compared with each other, under one label and under t % 64 labels,
so that every warp flushes mid-row after 65 536 tiles with its shared per-label accumulators near their 2^59 bound; and a long
session in which one (c, g) passes 2^64 in D1 and 2^128 in D2 only after thousands of accumulates, equal to that many times
the single call.

The rows are a 21.6 GB Form D tensor on the device, attached to a fresh engine in a process of its own (APO_K1_GRID is read
once per process)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import group_pair_fixtures as gf
import pair_fixtures as pf
import spread_fixtures as sf

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))

FLUSH_SCRIPT = r"""
import json, sys
import numpy as np
sys.path[:0] = [sys.argv[1], sys.argv[2]]
from importlib import import_module
import torch
import pair_fixtures as pf, spread_fixtures as sf
apo = import_module("senweaver-ide_b200")
T = 300_000_000
buf = torch.full((2, T, 9), float("nan"), dtype=torch.float32, device="cuda:0")
buf[0, :, 1] = sf.F32_BELOW_512
buf[1, :, 1] = -512.0
torch.cuda.synchronize()
e = apo.Engine(0)
try:
    e.set_weights(sf.w_one())
    e.candidate_refs_upload([1, 0])
    e.dims_attach(buf.data_ptr(), 2, T, T)
    G = int(sys.argv[3])
    e.record_groups_upload(np.tile(np.arange(G, dtype=np.uint8), T // G), G)
    r = e.score(2, 1, group_pairs=True)
    got = [[[int(p.ref), int(p.n), int(p.wins), int(p.losses), int(p.ties), p.sum, p.sum_sq, p.meanDiff.hex(), p.variance.hex()] for p in row]
           for row in r.group_pairs]
finally:
    e.close()
want = [pf.constant_pair(T // G, sf.F32_BELOW_512, -512.0, 1), pf.constant_pair(T // G, -512.0, sf.F32_BELOW_512, 0)]
want = [[[m["ref"], m["n"], m["wins"], m["losses"], m["ties"], m["D1"], m["D2"], m["meanDiff"].hex(), m["variance"].hex()]] * G for m in want]
print(json.dumps({"ok": got == want, "got": str(got)[:2000], "want": str(want)[:2000]}))
"""


@pytest.mark.parametrize("G", [1, 64])
def test_run_flush_at_one_cta_over_600M_evaluations(G):
    """one CTA of 8 warps over C = 2 rows of T = 3e8 (K1 on an attached tensor): ~73 000 tiles per warp, so every warp
    flushes mid-row after 65 536 tiles; at G = 1 the (c, 0) D1 ~ 2^90 and D2 ~ 2^152, at G = 64 (T divisible by 64) every
    label holds T / 64 positions"""
    env = dict(os.environ, APO_K1_GRID="1")
    p = subprocess.run([sys.executable, "-c", FLUSH_SCRIPT, ROOT, HERE, str(G)], env=env, capture_output=True, text=True, timeout=3000)
    assert p.returncode == 0, p.stderr[-4000:]
    out = json.loads(p.stdout.strip().splitlines()[-1])
    assert out["ok"], out


def test_long_session_past_2_64_and_2_128(engine, orc):
    """rows at fr = 1 and -1 (d = 2^53) of 1024 + 7 evaluations with a few nulls, label 1 on the last 5 and label 0 on the rest,
    accumulated 4500 times: in label 0 D1 passes 2^64 after a handful of accumulates and D2 passes 2^128 only after ~4000; every
    word of both labels equals 4500 times the single call's"""
    T, K = 1024 + 7, 4500
    d = np.stack([pf.rows(T, d1=np.float32(1.0)), pf.rows(T, d1=np.float32(-1.0))])
    d[0, 100] = np.nan
    d[1, T - 1] = np.nan
    lab, G = (np.arange(T) >= T - 5).astype(np.uint8), 2
    try:
        engine.set_weights(sf.w_one())
        engine.set_tuning(0x10)
        engine.dims_upload(d)
        engine.candidate_refs_upload([1, 0])
        engine.record_groups_upload(lab, G)
        one = gf.model(d, [1, 0], lab, G, sf.w_one())
        assert one[0][0]["D2"] * K > 2 ** 128 > one[0][0]["D2"] * (K // 2) and abs(one[0][0]["D1"]) * 8 > 2 ** 64
        engine.score_begin(2)
        for _ in range(K):
            engine.score_accumulate(0, group_pairs=True)
        res = engine.score_finish(2, 1, group_pairs=True)
        for c in range(2):
            for g in range(G):
                p, m = res.group_pairs[c][g], one[c][g]
                want = pf.pair_fields(m["ref"], K * m["n"], K * m["wins"], K * m["losses"], K * m["ties"], K * m["candOnly"], K * m["refOnly"],
                                      K * m["D1"], K * m["D2"])
                assert (p.sum, p.sum_sq, int(p.n), int(p.candOnly), int(p.refOnly)) == (want["D1"], want["D2"], want["n"], want["candOnly"],
                                                                                        want["refOnly"]), (c, g)
                assert (p.meanDiff.hex(), p.variance.hex(), p.stdErr.hex()) == (want["meanDiff"].hex(), want["variance"].hex(),
                                                                               want["stdErr"].hex()), (c, g)
    finally:
        engine.set_tuning(0)
        engine.set_weights(orc.weights())
