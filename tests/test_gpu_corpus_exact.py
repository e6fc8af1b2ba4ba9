"""Every corpus report bit for bit against the exact report of tests/exact_report.py, on the H100 (-m gpu).

The other corpus-report tests compare with oracle.report, which sums in sequential binary64 as the reference does: they allow
1e-12 on every sum and average, let a flag at a threshold fall either way, and check only the integers of saturating corpora.
Here every field of every report -- each sum and average rounded once from its exact fixed-point integer, each flag and
severity from that average, the NaNs -- must equal the exact report's bytes, with no tolerance and no waiver, on every host
that builds one:

- the resident corpus report: the corpus warp of K1 / K1q / K1r / K1r16 (TUNE_FORCE_FUSE), k_detect6_tiles (TUNE_NO_FUSE),
  the grid-stride k_detect6 (APO_K2_GRIDSTRIDE=1, in a subprocess) and a session; on the threshold fixtures, generated
  corpora of 1, 37, 1000 and 100 003 records, and the 36 M-record planted and saturating corpora of test_gpu_corpus_flush
  (with and without the digest);
- the digest built at load, through k_corpus_digest and inside K1h's one launch: the flagship fixtures, and the threshold
  fixtures padded past the digest's minimum size;
- the per-candidate corpus report: the 15 x 5 M Form R16 rows of test_gpu_corpus_flush resident, streamed and in reversed
  sessions, 8 of them as Form R, the threshold fixtures as rows, and the 128 x 5 M generated rollouts of
  examples/candidates_cost.py as R16 and as R (8 spread rows, against oracle/candidates.py's generator path);
- weights set after the load, one of them zero and the linspace(0.05, 0.45, 9) set, on the digest route (which recomputes
  every reward from its key), on k_detect6_tiles and on the per-candidate report."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import exact_report as xr
import flagship_fixtures as ff
import test_gpu_corpus_flush as flush
import test_gpu_count_route as cr
from test_gpu_candidates import boundary_records
from test_gpu_corpus_digest import _NoDigest
from test_gpu_flagship_edges import digest_case

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
BASES = (0, (1 << 40) + 8)
GEN = ((1, 5), (37, 0), (1000, 0), (100_003, 1 << 33))          # (T, idx_base) of the generated corpora
GEN_SEED = 0x5EED0003


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(autouse=True)
def restore(engine, orc):
    engine.set_tuning(0)
    yield
    engine.set_tuning(0)
    engine.set_weights(orc.weights())


def weight_sets(orc):
    w3 = orc.weights().copy()
    w3[3] = 0.0                                                     # d3 present but weightless
    d5_only = np.array([0.0] * 5 + [1.0] + [0.0] * 3)               # masks without d5 weigh 0: null rewards
    return {"d3_zero": w3, "d5_only": d5_only, "linspace": np.linspace(0.05, 0.45, 9)}


def as_report(apo, b):
    return apo.engine.CorpusReport.from_buffer_copy(bytes(b))


def corpus_case(name, sm):
    """(records, idx_base) of a named corpus: thr:<threshold fixture>, gen:<T>:<idx_base>, big:<kind>:<idx_base>"""
    kind, _, rest = name.partition(":")
    if kind == "thr":
        return {n: r for n, r, *_ in xr.threshold_fixtures()}[rest], 3
    a, b = rest.split(":")
    if kind == "gen":
        import oracle
        return oracle.gen_records(GEN_SEED, oracle.STREAM_CORPUS, 0, 1, int(b), int(a), 300, 8).reshape(-1), int(b)
    return flush.big_corpus(a, sm, int(b))[0], int(b)


SMALL = [f"thr:{n}" for n, *_ in xr.threshold_fixtures()] + [f"gen:{T}:{b}" for T, b in GEN]
BIG = [f"big:{k}:{b}" for k, b in (("saturating", BASES[1]), ("planted", 0), ("planted", BASES[1]), ("saturating", 0))]


# ------------------------------------------------------------------------------------------------ the resident corpus report
def check_hosts(apo, reps, want, what):
    for host, b in reps.items():
        xr.check_exact(as_report(apo, b), want, f"{what} {host}")


def test_small_corpora_every_scan_host(engine, orc, apo, sm_count):
    for name in SMALL:
        recs, base = corpus_case(name, sm_count)
        check_hosts(apo, flush.every_scan_host(engine, orc, apo, recs, base), xr.exact_report(recs, base), name)


@pytest.mark.parametrize("name", BIG)
def test_36M_corpus_every_scan_host(engine, orc, apo, sm_count, name):
    """the 36 M-record flush cases, scanned by every host (no digest), then with the digest the load builds taking over from
    the second reported call"""
    recs, base = corpus_case(name, sm_count)
    want = xr.exact_report(recs, base)
    check_hosts(apo, flush.every_scan_host(_NoDigest(engine, apo), orc, apo, recs, base), want, f"{name} scan")
    engine.set_tuning(0)
    check_hosts(apo, flush.every_scan_host(engine, orc, apo, recs, base), want, f"{name} digest")
    assert engine.debug_corpus_digest() is not None


GRIDSTRIDE_SCRIPT = r"""
import importlib, json, sys
sys.path[:0] = [sys.argv[1], sys.argv[2]]
import oracle
import test_gpu_corpus_exact as t
apo = importlib.import_module("senweaver-ide_b200")
e = apo.Engine(0)
e.dims_upload(oracle.gen_dims(0x5EED0C31, 0, 2, 0, 4096, 300, 2))
e.set_tuning(apo.TUNE_NO_FUSE | apo.TUNE_NO_CORPUS_DIGEST)
out = []
for name in json.loads(sys.argv[3]):
    recs, base = t.corpus_case(name, int(sys.argv[4]))
    e.corpus_upload(recs, base)
    out.append(bytes(e.score(2, 1, corpus=True).report).hex())
e.close()
print(json.dumps(out))
"""


def test_grid_stride_kernel(apo, sm_count):
    """k_detect6 (APO_K2_GRIDSTRIDE=1 is read once per process): the small corpora and two of the 36 M ones"""
    names = SMALL + BIG[:2]
    env = dict(os.environ, APO_K2_GRIDSTRIDE="1")
    p = subprocess.run([sys.executable, "-c", GRIDSTRIDE_SCRIPT, ROOT, HERE, json.dumps(names), str(sm_count)], env=env,
                       capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-3000:]
    got = json.loads(p.stdout.strip().splitlines()[-1])
    assert len(got) == len(names)
    for name, h in zip(names, got):
        recs, base = corpus_case(name, sm_count)
        xr.check_exact(as_report(apo, bytes.fromhex(h)), xr.exact_report(recs, base), f"{name} grid-stride")


# ------------------------------------------------------------------------------------------------ the digest built at load
@pytest.fixture
def k1h_dims(engine, apo):
    engine.set_tuning(apo.TUNE_TWIN_T)
    engine.dims_upload(cr.build())
    assert engine.debug_twin_h() is not None


def digest_cases():
    """(name, records, idx_base, kept) of the flagship fixtures"""
    yield "gate_small", ff.gate(ff.GATE_SMALL_T, 0), BASES[1], True
    yield "gate_small_over", ff.gate(ff.GATE_SMALL_T, 1), 0, False
    yield "gate_large", ff.gate(ff.GATE_LARGE_T, 0), 0, True
    yield "gate_invalid", ff.gate_invalid(ff.GATE_LARGE_T), BASES[1], True
    yield "no_valid", ff.no_valid(), 7, True
    yield "probe", ff.probe()[0], BASES[1], True
    for n in ff.FEW:
        yield f"few{n}", ff.few(n), BASES[1], True


def test_digest_flagship_fixtures(engine, apo, orc, k1h_dims):
    """K1h with the digest pass in its launch, K1t2 then k_corpus_digest, and the scan: the same bytes (digest_case), and
    those bytes the exact report"""
    for name, recs, base, kept in digest_cases():
        r = digest_case(engine, apo, orc, recs, base, kept)
        xr.check_exact(r.report, xr.exact_report(recs, base), name)


def test_digest_threshold_fixtures(engine, apo, orc, k1h_dims):
    """each threshold fixture followed by records without a reward, past the digest's minimum of 2^20 records"""
    for name, recs, *_ in xr.threshold_fixtures():
        big = xr.padded(recs, (1 << 20) + 5)
        r = digest_case(engine, apo, orc, big, BASES[1], kept=True)
        xr.check_exact(r.report, xr.exact_report(big, BASES[1]), name)


def test_weights_after_the_load_digest_and_scan(engine, apo, orc, k1h_dims):
    """a corpus digested under the default weights, then reported under each weight set: K1h's digest pass, k_corpus_digest
    after K1t2, and k_detect6_tiles"""
    recs = orc.gen_records(0x5EED0E01, orc.STREAM_CORPUS, 0, 1, 0, (1 << 21) + 3, 300).reshape(-1)
    engine.set_tuning(apo.TUNE_TWIN_T)
    engine.corpus_upload(recs, 11)
    for _ in range(2):
        engine.score(cr.C, 2, corpus=True)
    assert engine.debug_corpus_digest() is not None
    for wname, w in weight_sets(orc).items():
        engine.set_weights(w)
        want = xr.exact_report(recs, 11, w=w)
        for tname, flags in (("K1h", apo.TUNE_TWIN_T), ("k_corpus_digest", apo.TUNE_TWIN_T | apo.TUNE_NO_TWIN_H),
                             ("tiles", apo.TUNE_NO_FUSE | apo.TUNE_NO_CORPUS_DIGEST)):
            engine.set_tuning(flags)
            r = engine.score(cr.C, 2, corpus=True)
            assert tname != "K1h" or r.timing.launches == 1, wname
            xr.check_exact(r.report, want, f"{wname} {tname}")
        engine.set_weights(orc.weights())
    assert engine.debug_corpus_digest() is not None


# ------------------------------------------------------------------------------------------------ per-candidate corpus reports
def check_rows(reports, wants, what):
    assert len(reports) == len(wants)
    for c, (r, want) in enumerate(zip(reports, wants)):
        xr.check_exact(r, want, f"{what} row {c}")


def test_cand_corpus_threshold_rows_and_weights(engine, orc, apo):
    """the threshold fixtures as rows of Form R and R16 (padded to one length); boundary records under every weight set"""
    fixtures = xr.threshold_fixtures()
    L = max(len(r) for _, r, *_ in fixtures)
    rows = np.stack([xr.padded(r, L) for _, r, *_ in fixtures])
    wants = xr.exact_rows(rows, 0)
    engine.rollouts_upload(rows)
    check_rows(engine.score(len(rows), 1, source=apo.SRC_ROLLOUTS, candidate_corpus=True).candidate_corpus, wants, "R")
    engine.rollouts16_upload(apo.pack16(rows))
    check_rows(engine.score(len(rows), 1, source=apo.SRC_ROLLOUTS, candidate_corpus=True).candidate_corpus, wants, "R16")
    recs = boundary_records(orc, 3, 8_000, seed=3)
    for wname, w in weight_sets(orc).items():
        engine.set_weights(w)
        engine.rollouts_upload(recs)
        res = engine.score(3, 2, source=apo.SRC_ROLLOUTS, candidate_corpus=True)
        check_rows(res.candidate_corpus, xr.exact_rows(recs, 0, w=w), wname)


@pytest.fixture(scope="module")
def cc_rows(orc, sm_count):
    p16 = flush.cand_rows16(sm_count)
    return p16, [xr.exact_report(orc.unpack16(p16[c])) for c in range(flush.CC_C)]


def test_cand_corpus_15x5M_resident_streamed_reversed_and_r(engine, orc, apo, cc_rows):
    p16, wants = cc_rows
    C = flush.CC_C
    engine.rollouts16_upload(p16)
    check_rows(engine.score(C, 4, source=apo.SRC_ROLLOUTS, candidate_corpus=True).candidate_corpus, wants, "resident")
    check_rows(engine.score_host_records(p16, 4, candidate_corpus=True).candidate_corpus, wants, "streamed")
    cuts = [0, 1_048_576, 2_000_000, 2_000_004, 4_999_000, flush.CC_T]
    engine.score_begin(C)
    for a, b in reversed(list(zip(cuts, cuts[1:]))):
        engine.score_accumulate(0, source=apo.SRC_ROLLOUTS, first=a, count=b - a, candidate_corpus=True)
    check_rows(engine.score_finish(C, 4, candidate_corpus=True).candidate_corpus, wants, "reversed windows")
    engine.score_begin(C)
    for c0 in (8, 0):                                                    # candidate chunks in reverse, each in reversed windows
        engine.rollouts16_upload(p16[c0:c0 + 8])
        engine.score_accumulate(c0, source=apo.SRC_ROLLOUTS, first=3_000_000, count=0, candidate_corpus=True)
        engine.score_accumulate(c0, source=apo.SRC_ROLLOUTS, first=0, count=3_000_000, candidate_corpus=True)
    check_rows(engine.score_finish(C, 4, candidate_corpus=True).candidate_corpus, wants, "reversed chunks")
    r32 = orc.unpack16(p16[:8])
    engine.rollouts_upload(r32)
    del r32
    check_rows(engine.score(8, 2, source=apo.SRC_ROLLOUTS, candidate_corpus=True).candidate_corpus, wants[:8], "Form R")


def test_cand_corpus_generated_128x5M_r16_and_r(orc, apo):
    """the rollout legs of examples/candidates_cost.py: seed 0x5EED0003, 128 x 5 M, 8 rows spread over C.  On an engine of
    its own, closed at the end: an engine's buffers only grow, and the 20 GB of Form R rows would otherwise stay resident
    in the session's engine and crowd the later full-size tests"""
    seed, C, T = GEN_SEED, 128, 5_000_000
    picks = [int(x) for x in np.linspace(0, C - 1, 8).round()]
    wants = xr.exact_generated(seed, picks, T)
    e = apo.Engine(0)
    try:
        for form, load in (("R16", e.rollouts16_generate), ("R", e.rollouts_generate)):
            load(seed, 0, C, 0, T, 300)
            cc = e.score(C, 4, source=apo.SRC_ROLLOUTS, candidate_corpus=True).candidate_corpus
            check_rows([cc[c] for c in picks], wants, form)
    finally:
        e.close()
