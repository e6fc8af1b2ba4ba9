"""The flagship step on a joined communicator (-m gpu; a world skips when the node has fewer GPUs): every rank holds the
Form T copy with its per-row dictionary counts over its shard of the rows' evaluations and a corpus shard of at least
2^20 + 17 records, so the second reported call builds a digest on every rank and the third runs K1h, the digest pass and the
peer-memory join in one launch -- the path bench.py takes at N = 2 and N = 4.  Every rank's scores, top-K, joined integers
and report bytes must equal the unsharded single-GPU call's and the same ranks' with TUNE_NO_CORPUS_DIGEST (the scan), and
the report the oracle's; in the planted case the first three examples of every pattern straddle a shard boundary, so they
come from two ranks' example slots."""
import os
import sys
from importlib import import_module

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import corpus_fixtures as cf
from test_gpu_candidate_corpus import check_oracle

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
C, K, SEED = 16, 4, 0x5EEDF109
T_RANK = 500_000                         # evaluations per row and rank: few enough distinct ones for the counts' gate
TC_RANK = (1 << 20) + 17                 # corpus records per rank: at least the digest's minimum


def planted(Tc, boundary):
    """corpus_fixtures.planted with every pattern's hits late, plus hits at boundary - 1, boundary and boundary + 1"""
    extra = {p: [boundary - 1, boundary, boundary + 1] for p in range(6)}
    return cf.planted(Tc, kinds=(0,) * 6, extra=extra)


def calls(eng, flags):
    eng.set_tuning(flags)
    rs = [eng.score(C, K, corpus=True) for _ in range(3)]
    return rs[-1]


def worker(rank, world, uid_path, out_dir, case):
    sys.path[:0] = [ROOT, HERE]
    pkg = import_module("senweaver-ide_b200")
    torch.cuda.set_device(rank)
    eng = pkg.Engine(rank)
    eng.comm_init(world, rank, open(uid_path, "rb").read())
    eng.set_tuning(pkg.TUNE_TWIN_T)
    first, last = pkg.sharding.shard_range(T_RANK * world, world, rank)
    eng.dims_generate(SEED, 0, C, first, last - first, 300)
    held = eng.debug_twin_h() is not None
    Tc = TC_RANK * world
    c0, c1 = pkg.sharding.shard_range(Tc, world, rank)
    if case == "planted":
        recs, _, _ = planted(Tc, pkg.sharding.shard_range(Tc, world, 1)[0])
        eng.corpus_upload(recs[c0:c1], c0)
    else:
        eng.corpus_generate(SEED, c0, c1 - c0, 300)
    r = calls(eng, pkg.TUNE_TWIN_T)
    digest = eng.debug_corpus_digest() is not None
    sums, counts = eng.debug_partials(C)
    scan = calls(eng, pkg.TUNE_TWIN_T | pkg.TUNE_NO_CORPUS_DIGEST)
    np.savez(os.path.join(out_dir, f"r{rank}.npz"), scores=r.scores, topk=r.topk, counts=np.array(counts),
             sums=np.array([str(s) for s in sums]), report=np.frombuffer(bytes(r.report), np.uint8),
             scan_report=np.frombuffer(bytes(scan.report), np.uint8), scan_scores=scan.scores, scan_topk=scan.topk,
             launches=np.array([r.timing.launches]), held=np.array([held, digest]), mode=np.array([eng.comm_join_mode()]))
    eng.close()


@pytest.mark.parametrize("case", ["generated", "planted"])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_k1h_digest_and_join_in_one_launch(tmp_path, engine, orc, apo, world, case):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    uid_path = tmp_path / "uid.bin"
    uid_path.write_bytes(apo.Engine.comm_unique_id())
    mp.spawn(worker, args=(world, str(uid_path), str(tmp_path), case), nprocs=world, join=True)
    Tc = TC_RANK * world
    engine.set_tuning(apo.TUNE_TWIN_T)
    try:
        engine.dims_generate(SEED, 0, C, 0, T_RANK * world, 300)
        if case == "planted":
            recs, _, want = planted(Tc, apo.sharding.shard_range(Tc, world, 1)[0])
            engine.corpus_upload(recs, 0)
            ref = orc.report(recs, nthreads=16)
        else:
            engine.corpus_generate(SEED, 0, Tc, 300)
            ref = orc.report_generated(SEED, 0, Tc)
        single = calls(engine, apo.TUNE_TWIN_T)
        rsums, rcounts = engine.debug_partials(C)
    finally:
        engine.set_tuning(0)
    check_oracle(apo, single.report, ref)
    if case == "planted":
        cf.check_designed(single.report, want)
    for r in range(world):
        z = np.load(tmp_path / f"r{r}.npz")
        assert list(z["held"]) == [True, True] and z["mode"][0] == 2 and z["launches"][0] == 1, r
        assert [int(s) for s in z["sums"]] == rsums and list(z["counts"]) == rcounts
        assert np.array_equal(z["scores"], single.scores) and np.array_equal(z["topk"], single.topk)
        assert np.array_equal(z["scan_scores"], single.scores) and np.array_equal(z["scan_topk"], single.topk)
        assert z["report"].tobytes() == z["scan_report"].tobytes() == bytes(single.report), r
