"""Small end-to-end exercise of every kernel, meant to run under compute-sanitizer:

    compute-sanitizer --tool memcheck  python tests/sanitize_smoke.py
    compute-sanitizer --tool racecheck python tests/sanitize_smoke.py
    compute-sanitizer --tool synccheck python tests/sanitize_smoke.py

(also a plain script: prints OK when every result matches the oracle)."""
import importlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import oracle as orc  # noqa: E402

pkg = importlib.import_module("senweaver-ide_b200")
e = pkg.Engine(0)
C, T, seed = 5, 7001, 0x5EED00AA
dims = orc.gen_dims(seed, 0, C, 0, T, 400, 4)
recs = orc.gen_records(seed, orc.STREAM_CORPUS, 0, 1, 0, T, 400, 4).reshape(-1)
roll = orc.gen_records(seed, orc.STREAM_ROLLOUT, 0, C, 0, T, 400, 4)
exp = orc.score_dims_fx(dims)
e.dims_upload(dims)
e.corpus_upload(recs)
for v in range(5):
    r = e.score(C, 3, corpus=True, variant=v)
    assert e.debug_partials(C) == exp
ref = orc.report(recs)
assert [r.report.pat[p].count for p in range(6)] == [ref.pat[p].count for p in range(6)]
e.set_tuning(pkg.TUNE_FORCE_FUSE)             # the corpus scan inside the scoring launch (K1, then K1q / K1r below)
r = e.score(C, 3, corpus=True)
assert r.timing.launches == 1 and e.debug_partials(C) == exp
assert [r.report.pat[p].count for p in range(6)] == [ref.pat[p].count for p in range(6)] and list(r.report.pat[0].examples) == list(ref.pat[0].examples)
e.score(C, 2, first=1000, count=3001)
assert e.debug_partials(C) == orc.score_dims_fx(dims[:, 1000:4001])
e.dims_compact()
for v in range(7):                           # 0 mixed lookup (default), 1-3 tile shapes, 4 product tables only, 5-6 more fp32 lookups
    e.score(C, 3, variant=v)
    assert e.debug_partials(C) == exp
assert np.array_equal(np.nan_to_num(e.dims_download(2, 0, T), nan=7), np.nan_to_num(dims[2], nan=7))
e.dims_generate_compact(seed, 0, C, 0, T, 400)
r = e.score(C, 1, corpus=True)
assert r.timing.launches == 1 and e.debug_partials(C) == exp and r.report.bad == ref.bad
e.rollouts_upload(roll)
e.score(C, 2, source=1)
assert e.debug_partials(C) == orc.score_records_fx(roll)
e.rollouts16_upload(pkg.pack16(roll))
r = e.score(C, 2, source=1, corpus=True)
assert r.timing.launches == 1 and e.debug_partials(C) == orc.score_records_fx(roll) and r.report.bad == ref.bad
e.set_tuning(0)
e.score_host(dims, 2)
assert e.debug_partials(C) == exp
e.score_host_records(pkg.pack16(roll), 2)
assert e.debug_partials(C) == orc.score_records_fx(roll)
d, m, f = e.reward_batch(recs[:500])
d1, m1, f1 = e.reward_batch(recs[:3])                 # zero-copy single-trace path (kernel reads / writes page-locked host memory)
assert np.array_equal(f1, f[:3], equal_nan=True)
# round-2 kernels: stand-alone corpus scan as TMA tiles (>= 8192 records), the packed / compact wire formats, their export
big = orc.gen_records(seed, orc.STREAM_CORPUS, 0, 1, 0, 20_000, 300, 4).reshape(-1)
e.corpus_upload(big)
e.dims_upload(dims)
e.score_begin(C)
e.score_accumulate(0)
r = e.score_finish(C, 3, corpus=True)                 # k_detect6_tiles + fused K3
refb = orc.report(big)
assert r.report.bad == refb.bad and [r.report.pat[p].count for p in range(6)] == [refb.pat[p].count for p in range(6)]
assert list(r.report.pat[2].examples) == list(refb.pat[2].examples)
pc, pd, book, d2book = pkg.packed_encode_host(dims, nthreads=2)
e.score_host_packed(pc, pd, book, d2book, 2, corpus=True)         # k_unpack_p + K1q
assert e.debug_partials(C) == exp
q8, d2, li, book2 = pkg.compact_encode_host(dims, nthreads=2)
e.score_host_compact(q8, d2, li, book2, 2)
assert e.debug_partials(C) == exp
e.dims_upload_compact(dims)
a, b = e.dims_packed_download(1, 0, T)                            # k_collect_d2 + k_pack_p
assert np.array_equal(a, pc[1]) and np.array_equal(b, pd[1])
# Form T: k_tuple_values + K1t, full tiles (8192 evaluations) and ragged row ends, streamed and resident
dt = orc.gen_dims(seed, 0, 3, 0, 2 * 8192 + 77, 400, 4)
pt, pdt, bkt, d2t = pkg.packed_encode_host(dt, nthreads=2)
tl, th, tbook = pkg.tuple_encode_host(pt, pdt, nthreads=2)
e.score_host_tuples(tl, th, tbook, bkt, d2t, 2, corpus=True)
assert e.debug_partials(3) == orc.score_dims_fx(dt)
e.tuples_upload(tl, th, tbook, bkt, d2t)
e.score(3, 2, source=pkg.SRC_TUPLES, first=8, count=8192 + 100)
assert e.debug_partials(3) == orc.score_dims_fx(dt[:, 8:8192 + 108])
# Form T, hand-built (tests/tuple_fixtures.py): the largest dictionary (2^24 - 1 entries), indices with every high byte
sys.path.insert(0, os.path.join(ROOT, "tests"))
import tuple_fixtures as tfx  # noqa: E402
tbx, bkx, d2x = tfx.dictionary(tfx.TUPLES_MAX), tfx.codebook(), tfx.d2book()
ix = tfx.hi_byte_groups(tfx.TUPLES_MAX, 2, 2 * 8192 + 77)
assert len(np.unique(ix >> 16)) == 256
wx = tfx.expected(ix, *tfx.entry_fx(tbx, bkx, d2x))
e.score_host_tuples(*tfx.planes(ix), tbx, bkx, d2x, 1)
assert e.debug_partials(2) == wx
e.tuples_upload(*tfx.planes(ix), tbx, bkx, d2x)
e.score(2, 1, source=pkg.SRC_TUPLES)
assert e.debug_partials(2) == wx
e.tuples_upload(tl, th, tbook, bkt, d2t)                          # the generated tensor again, for the breakdown below
# per-candidate breakdown (k_cand_breakdown + k_cand_report) on every record source, and the per-candidate corpus reports
# (k_cand_corpus + k_cand_corpus_report) on the two that carry record fields
from oracle import candidates as oc  # noqa: E402
oc.build()
dref = [(d["bad"], d["badExamples"]) for d in oc.cand_dims(dt)]
for run in (lambda: e.score(3, 1, source=pkg.SRC_TUPLES, candidates=True),
            lambda: e.score_host_tuples(tl, th, tbook, bkt, d2t, 1, candidates=True),
            lambda: e.score_host_packed(pt, pdt, bkt, d2t, 1, candidates=True),
            lambda: e.score_host(dt, 1, candidates=True)):
    assert [(b.bad, list(b.badExamples)) for b in run().candidates] == dref
e.dims_upload(dt)
assert [(b.bad, list(b.badExamples)) for b in e.score(3, 1, candidates=True).candidates] == dref
e.dims_upload_compact(dt)
assert [(b.bad, list(b.badExamples)) for b in e.score(3, 1, candidates=True).candidates] == dref
rref = [(d["bad"], d["badExamples"]) for d in oc.cand_records(roll)]
e.rollouts_upload(roll)
assert [(b.bad, list(b.badExamples)) for b in e.score(C, 2, source=1, candidates=True).candidates] == rref
cc = e.score(C, 2, source=1, candidate_corpus=True).candidate_corpus
assert [bytes(x) for x in e.score_host_records(roll, 2, candidate_corpus=True).candidate_corpus] == [bytes(x) for x in cc]
assert [(b.bad, list(b.badExamples)) for b in e.score_host_records(roll, 2, candidates=True).candidates] == rref
for c in range(C):
    rc = orc.report(roll[c])
    assert cc[c].bad == rc.bad and [list(cc[c].pat[p].examples) for p in range(6)] == [list(rc.pat[p].examples) for p in range(6)]
r16 = pkg.pack16(roll)
rref = [(d["bad"], d["badExamples"]) for d in oc.cand_records(orc.unpack16(r16))]
e.rollouts16_upload(r16)
assert [(b.bad, list(b.badExamples)) for b in e.score(C, 2, source=1, candidates=True).candidates] == rref
assert [(b.bad, list(b.badExamples)) for b in e.score_host_records(r16, 2, candidates=True).candidates] == rref
cc = e.score(C, 2, source=1, candidate_corpus=True).candidate_corpus
assert [bytes(x) for x in e.score_host_records(r16, 2, candidate_corpus=True).candidate_corpus] == [bytes(x) for x in cc]
assert [cc[c].pat[1].count for c in range(C)] == [orc.report(orc.unpack16(r16[c])).pat[1].count for c in range(C)]
for Cn in ((3, 1500, 3000) if not os.environ.get("SMOKE_NO_MANY_CANDIDATES") else ()):       # counting top-K (<= 2048 keys in shared memory) and the radix select
    e.dims_generate(seed, 0, Cn, 0, 64, 300)
    r = e.score(Cn, min(Cn, 40))
    sc = r.scores
    order = sorted(range(Cn), key=lambda c: (-sc[c], c))[:min(Cn, 40)]
    assert list(r.topk) == order
e.dims_generate(seed, 0, 2, 0, 300, 300)
e.rollouts_generate(seed, 0, 2, 0, 300, 300)
e.rollouts16_generate(seed, 0, 2, 0, 300, 300)
e.corpus_generate(seed, 0, 300, 300)
e.close()
print("OK")
