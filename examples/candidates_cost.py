"""What the per-candidate breakdown (APO_SCORE_CANDIDATES) costs: the flagged scoring step beside the plain one, in the
same process, alternating, on the configs[2] workload (256 x 5 M) resident as Form D, Form Q and Form T, and on 128 x 5 M
Form R16 rollouts.  Every leg carries a parity block: the full breakdown of 8 candidates spread over C, over the whole
record axis, against the CPU oracle's generator path (integers, first-three examples and every binary64 field).

The rollout legs (R16, and R = the same rollouts as 32-byte records) also time the step with the per-candidate corpus
reports (APO_SCORE_CANDIDATE_CORPUS), alternating plain / candidates / candidate_corpus, and add a second parity block: the
corpus report of the same 8 candidates against the exact report of their generated rows (tests/exact_report.py: every
field bit for bit, each sum rounded once from its exact fixed-point integer).  Beside it, parity_corpus_seq keeps the older
comparison with oracle.report (binary64 sums to 1e-12, the oracle summing per-thread slices in sequential binary64) and lists
the fields that fail it.

Every leg also times the step with the per-candidate extremes (APO_SCORE_CANDIDATE_EXTREMES) in the same alternation.  On the
fp32 legs its parity block is the lists of two of the 8 candidates against the model of tests/extremes_fixtures.py over the
generated rows (positions and rewards bit for bit); on the rollout legs every list holds min(32, counts[c]) entries and R16
and R give the same bytes.  Leg W is Form D through its Form W copy (the Form T copy held beside it is switched off), leg
FALL is 64 x 1 M strictly falling rows through K1, where every group of 32 evaluations runs the extremes' merge network.

Every leg also times the step with the per-candidate group scores (APO_SCORE_CANDIDATE_GROUPS) in the same alternation, under
five label planes: G = 1, and G = 5 and 64 both as contiguous runs (t * G // T) and as a new label on every record (t % G).
The labels are uploaded before each such step, outside its timing.  On the fp32 legs the parity block is the group scores
of two of the 8 candidates against the model of tests/group_fixtures.py over the generated rows (every field bit for bit);
on the rollout legs the non-null counts of every candidate's groups add up to counts[c], and R16 and R give the same bytes.

Every leg also times the step with the per-candidate reward spread (APO_SCORE_CANDIDATE_SPREAD) in the same alternation.  Its
parity block holds n and S1 of every candidate against apo_debug_partials (and mean against scores[c]); on the fp32 legs also
the spreads of two of the 8 candidates against the exact model of tests/spread_fixtures.py over the generated rows (every
field bit for bit), and on the rollout legs R16 and R give the same bytes.

Every leg also times the step with the paired comparison (APO_SCORE_CANDIDATE_PAIRS) in the same alternation, under refs
shaped like a beam: each candidate names the first candidate of its block of 5, which names none (the refs are uploaded once
per leg, outside the timing).  Its parity block holds the invariants of tests/pair_fixtures.py on every candidate (n + candOnly
and n + refOnly against counts[], wins + losses + ties == n, nothing for a candidate without a reference); on the fp32 legs
also the pairs of two candidates against the exact model of tests/pair_fixtures.py over the generated rows (every field bit
for bit), and on the rollout legs R16 and R give the same bytes.

Every leg also times the paired comparison per record group (APO_SCORE_CANDIDATE_GROUP_PAIRS) under the same refs and each of
the groups steps' label planes (gp_<plane>), in the same alternation.  Its parity block holds, on every candidate, the
invariants of tests/group_pair_fixtures.py against the pairs step's pairs (summed over the labels every integer field, the
same ref in every group); on the fp32 legs also two candidates' groups against the exact model of that module over the
generated rows, and on the rollout legs R16 and R give the same bytes.

    python examples/candidates_cost.py [--steps 10] [--legs D,W,Q,T,R16,R,FALL] [--out FILE.json]

Prints one JSON object; the card name and power limit are read in the same run (nvidia-smi query)."""
import argparse
import json
import os
import struct
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:       # the numbers are still printed; without the card line they are not comparable
        return f"unknown ({ex})"


def bits(x):
    return struct.pack("<d", x)


def same(r, d):
    if (r.total, r.good, r.bad, r.none, r.withReward) != (d["total"], d["good"], d["bad"], d["none"], d["withReward"]):
        return False
    if (bits(r.goodRate), bits(r.rewardSum), bits(r.avgReward)) != (bits(d["goodRate"]), bits(d["rewardSum"]), bits(d["avgReward"])):
        return False
    for i in range(9):
        a, b = r.dim[i], d["dim"][i]
        if (bits(a.sum), a.count, bits(a.avg), a.low_flag, a.low_severity, a.sugg_flag, a.sugg_priority) != \
           (bits(b["sum"]), b["count"], bits(b["avg"]), b["low_flag"], b["low_severity"], b["sugg_flag"], b["sugg_priority"]):
            return False
    return list(r.badExamples) == d["badExamples"]


def lists(x):
    return (int(x.n), list(x.lowest), list(x.highest), np.array(x.lowestReward).tobytes(), np.array(x.highestReward).tobytes())


def model_lists(m):
    return (m["n"], m["lowest"], m["highest"], np.array(m["lowestReward"]).tobytes(), np.array(m["highestReward"]).tobytes())


def extremes_parity(res, ref_ext):
    """ref_ext: {candidate: model lists}; without models, every list holds min(32, counts[c]) entries"""
    if ref_ext is None:
        return {"equal": all(int(x.n) == min(32, int(n)) for x, n in zip(res.extremes, res.counts)), "check": "n == min(32, counts)"}
    ok = {c: lists(res.extremes[c]) == model_lists(m) for c, m in ref_ext.items()}
    return {"candidates": list(ok), "equal": all(ok.values())}


def label_sets(T):
    """name -> (labels, G): G = 1, and G = 5 / 64 as contiguous runs and as a new label on every record"""
    t = np.arange(T, dtype=np.int64)
    out = {"groups_g1": (np.zeros(T, np.uint8), 1)}
    for G in (5, 64):
        out[f"groups_g{G}_runs"] = ((t * G) // T).astype(np.uint8), G
        out[f"groups_g{G}_every"] = (t % G).astype(np.uint8), G
    return out


def group_rows(x):
    return [[(s.total, s.good, s.bad, bits(s.goodRate), s.withReward, bits(s.rewardSum), bits(s.avgReward)) for s in row] for row in x]


def model_rows(m):
    return [[(s["total"], s["good"], s["bad"], bits(s["goodRate"]), s["withReward"], bits(s["rewardSum"]), bits(s["avgReward"]))
             for s in row] for row in m]


def groups_parity(last, sets, ref_grp):
    """ref_grp: {candidate: {set name: model row}}; without models, every candidate's groups add up to counts[c]"""
    out = {}
    for k in sets:
        r = last[k]
        sums = all(sum(s.withReward for s in row) == int(n) for row, n in zip(r.groups, r.counts))
        if ref_grp is None:
            out[k] = {"equal": sums, "check": "sum of withReward == counts"}
        else:
            ok = {c: group_rows([r.groups[c]]) == model_rows([m[k]]) for c, m in ref_grp.items()}
            out[k] = {"candidates": list(ok), "equal": all(ok.values()) and sums}
    return out


def spread_row(s):
    return (int(s.n), s.sum, s.sum_sq, bits(s.mean), bits(s.rewardSumSq), bits(s.variance), bits(s.stdDev), bits(s.stdErr))


def model_spread(m):
    return (m["n"], m["S1"], m["S2"], bits(m["mean"]), bits(m["rewardSumSq"]), bits(m["variance"]), bits(m["stdDev"]), bits(m["stdErr"]))


def spread_parity(eng, res, ref_spr):
    """n / S1 of every candidate against the scoring call's partials (every step of a leg sums the same integers), mean against
    scores[c]; ref_spr: {candidate: model spread}"""
    sums, counts = eng.debug_partials(len(res.spread))
    every = all((s.sum, int(s.n)) == (sums[c], counts[c]) and (s.n == 0 or bits(s.mean) == bits(res.scores[c]))
                for c, s in enumerate(res.spread))
    out = {"n_s1_every_candidate": every}
    if ref_spr:
        ok = {c: spread_row(res.spread[c]) == model_spread(m) for c, m in ref_spr.items()}
        out.update({"candidates": list(ok), "per_candidate": ok})
        every = every and all(ok.values())
    out["equal"] = every
    return out


def spread_block(eng, last, med, ref_spr):
    return {"spread_ms_median": round(med["spread"], 3), "spread_ratio": round(med["spread"] / med["plain"], 3),
            "spread_same_scores": last["spread"].scores.tobytes() == last["plain"].scores.tobytes()
                                  and last["spread"].topk.tobytes() == last["plain"].topk.tobytes(),
            "parity_spread": spread_parity(eng, last["spread"], ref_spr)}


def beam_refs(C):
    """each candidate names the first candidate of its block of 5 (a parent and its four children), which names none"""
    import pair_fixtures as pf
    return np.array([pf.NONE if c % 5 == 0 else c - c % 5 for c in range(C)], np.uint32)


def pair_row(p):
    return (int(p.ref), int(p.n), int(p.wins), int(p.losses), int(p.ties), int(p.candOnly), int(p.refOnly), p.sum, p.sum_sq,
            bits(p.meanDiff), bits(p.variance), bits(p.stdDev), bits(p.stdErr))


def model_pair(m):
    return (m["ref"], m["n"], m["wins"], m["losses"], m["ties"], m["candOnly"], m["refOnly"], m["D1"], m["D2"], bits(m["meanDiff"]),
            bits(m["variance"]), bits(m["stdDev"]), bits(m["stdErr"]))


def pairs_parity(res, ref_pair):
    """the invariants on every candidate against the call's counts; ref_pair: {candidate: model pair}"""
    import pair_fixtures as pf
    try:
        pf.invariants(res.pairs, [int(x) for x in res.counts])
        every = True
    except AssertionError:
        every = False
    out = {"invariants_every_candidate": every}
    if ref_pair:
        ok = {c: pair_row(res.pairs[c]) == model_pair(m) for c, m in ref_pair.items()}
        out.update({"candidates": list(ok), "per_candidate": ok})
        every = every and all(ok.values())
    out["equal"] = every
    return out


def pairs_block(last, med, ref_pair):
    return {"pairs_ms_median": round(med["pairs"], 3), "pairs_ratio": round(med["pairs"] / med["plain"], 3),
            "pairs_same_scores": last["pairs"].scores.tobytes() == last["plain"].scores.tobytes()
                                 and last["pairs"].topk.tobytes() == last["plain"].topk.tobytes(),
            "parity_pairs": pairs_parity(last["pairs"], ref_pair)}


def group_pairs_parity(last, gsets, ref_gpair):
    """the invariants on every candidate against the pairs step's pairs (the same refs and rows); ref_gpair: {candidate: {set
    name: model row [G]}}"""
    import group_pair_fixtures as gpf
    out = {}
    for k, (lab, G) in gsets.items():
        try:
            gpf.invariants(last[k].group_pairs, last["pairs"].pairs, G)
            every = True
        except AssertionError:
            every = False
        ok = {c: [pair_row(x) for x in last[k].group_pairs[c]] == [model_pair(m) for m in rows[k[3:]]] for c, rows in (ref_gpair or {}).items()}
        out[k] = {"invariants_every_candidate": every, "per_candidate": ok, "equal": every and all(ok.values())}
    return {"sets": out, "equal": all(v["equal"] for v in out.values())}


def group_pairs_block(last, med, gsets, ref_gpair):
    return {"group_pairs_ms_median": {k: round(med[k], 3) for k in gsets},
            "group_pairs_ratio": {k: round(med[k] / med["plain"], 3) for k in gsets},
            "group_pairs_vs_pairs": {k: round(med[k] / med["pairs"], 3) for k in gsets},
            "group_pairs_same_scores": all(last[k].scores.tobytes() == last["plain"].scores.tobytes()
                                           and last[k].topk.tobytes() == last["plain"].topk.tobytes() for k in gsets),
            "parity_group_pairs": group_pairs_parity(last, gsets, ref_gpair)}


def timed(eng, C, K, steps, score_kw, kinds, sets):
    """median / min of every kind of step, alternating; a group step first uploads its labels (outside the timing)"""
    times = {k: [] for k in kinds}

    def one(k, kw):
        if k in sets:
            eng.record_groups_upload(*sets[k])
        t0 = time.perf_counter(); r = eng.score(C, K, **kw, **score_kw); times[k].append(time.perf_counter() - t0)
        return r

    for _ in range(2):                                          # warm every shape
        for k, kw in kinds.items():
            one(k, kw)
    for v in times.values():
        v.clear()
    last = {}
    for _ in range(steps):                                      # alternate: drift and other tenants hit all alike
        for k, kw in kinds.items():
            last[k] = one(k, kw)
    return last, times, {k: float(np.median(v)) * 1e3 for k, v in times.items()}


def groups_block(last, med, sets, ref_grp):
    return {"groups_ms_median": {k: round(med[k], 3) for k in sets}, "groups_ratio": {k: round(med[k] / med["plain"], 3) for k in sets},
            "groups_same_scores": all(last[k].scores.tobytes() == last["plain"].scores.tobytes()
                                      and last[k].topk.tobytes() == last["plain"].topk.tobytes() for k in sets),
            "parity_groups": groups_parity(last, sets, ref_grp)}


def leg(eng, C, K, steps, score_kw, ref, picks, ref_ext=None, sets=None, ref_grp=None, ref_spr=None, ref_pair=None, ref_gpair=None):
    """plain / candidates / extremes / groups / spread / pairs / group_pairs steps, alternating (ref None: the breakdown is not
    timed)"""
    sets = sets or {}
    gsets = {f"gp_{k}": v for k, v in sets.items()}                 # the per-group pairs under each label plane
    kinds = {"plain": {}, "extremes": {"extremes": True}, "spread": {"spread": True}, "pairs": {"pairs": True}}
    eng.candidate_refs_upload(beam_refs(C))
    if ref is not None:
        kinds["candidates"] = {"candidates": True}
    kinds.update({k: {"groups": True} for k in sets})
    kinds.update({k: {"group_pairs": True} for k in gsets})
    last, times, med = timed(eng, C, K, steps, score_kw, kinds, {**sets, **gsets})
    out = {"plain_ms_median": round(med["plain"], 3), "extremes_ms_median": round(med["extremes"], 3),
           "extremes_ratio": round(med["extremes"] / med["plain"], 3), "min_ms": {k: round(min(v) * 1e3, 3) for k, v in times.items()},
           "launches": {k: int(r.timing.launches) for k, r in last.items()},
           "same_scores": last["extremes"].scores.tobytes() == last["plain"].scores.tobytes()
                          and last["extremes"].topk.tobytes() == last["plain"].topk.tobytes(),
           "parity_extremes": extremes_parity(last["extremes"], ref_ext)}
    out.update(groups_block(last, med, sets, ref_grp))
    out.update(spread_block(eng, last, med, ref_spr))
    out.update(pairs_block(last, med, ref_pair))
    out.update(group_pairs_block(last, med, gsets, ref_gpair))
    if ref is not None:
        r = last["candidates"]
        ok = [same(r.candidates[c], d) for c, d in zip(picks, ref)]
        out.update({"flagged_ms_median": round(med["candidates"], 3), "ratio": round(med["candidates"] / med["plain"], 3),
                    "parity": {"candidates": picks, "equal": all(ok), "per_candidate": ok,
                               "bad_examples": [list(r.candidates[c].badExamples) for c in picks]}})
    return out


def seq_corpus_diff(r, ref):
    """apo_corpus_report against oracle.report, the comparison of tests/test_gpu_parity.py check_report: integers, flags,
    examples and severities exactly, binary64 sums and averages to 1e-12 (the oracle sums in sequential binary64, merging
    per-thread slices).  Returns the fields that fail it, with both values."""
    close = lambda a, b: abs(a - b) <= 1e-12 * max(1.0, abs(b))
    out = []

    def need(ok, name, a, b):
        if not ok:
            out.append([name, a, b] + ([abs(a - b)] if isinstance(a, float) else []))

    for f in ("total", "good", "bad", "none", "withReward", "goodRate", "toolCalls", "toolSucc", "toolFail"):
        need(getattr(r, f) == getattr(ref, f), f, getattr(r, f), getattr(ref, f))
    for m in range(5):
        need(list(r.byMode[m]) == list(ref.byMode[m]), f"byMode[{m}]", list(r.byMode[m]), list(ref.byMode[m]))
        need(r.byModeGoodRate[m] == ref.byModeGoodRate[m], f"byModeGoodRate[{m}]", r.byModeGoodRate[m], ref.byModeGoodRate[m])
    if ref.withReward:
        need(close(r.avgReward, ref.avgReward), "avgReward", r.avgReward, ref.avgReward)
    for i in range(9):
        a, b = r.dim[i], ref.dim[i]
        need(a.count == b.count, f"dim[{i}].count", a.count, b.count)
        need(close(a.sum, b.sum), f"dim[{i}].sum", a.sum, b.sum)
        need(close(a.avg, b.avg), f"dim[{i}].avg", a.avg, b.avg)
        for f in ("low_flag", "sugg_flag"):
            need(getattr(a, f) == getattr(b, f), f"dim[{i}].{f}", getattr(a, f), getattr(b, f))
    for p in range(6):
        a, b = r.pat[p], ref.pat[p]
        need((a.count, a.flag, list(a.examples)) == (b.count, b.flag, list(b.examples)), f"pat[{p}]",
             [a.count, a.flag, list(a.examples)], [b.count, b.flag, list(b.examples)])
        need(not b.flag or a.severity == b.severity, f"pat[{p}].severity", a.severity, b.severity)
    return out


def parity_block(picks, diffs):
    return {"candidates": picks, "equal": not any(diffs), "per_candidate": [not d for d in diffs],
            "differing": {str(c): d for c, d in zip(picks, diffs) if d}}


def corpus_leg(eng, C, K, steps, score_kw, ref, picks, ref_corpus, sets):
    """plain / candidates / candidate_corpus / extremes / groups / spread / pairs / group_pairs steps, alternating, with the
    parity blocks"""
    kinds = {"plain": {}, "candidates": {"candidates": True}, "candidate_corpus": {"candidate_corpus": True}, "extremes": {"extremes": True},
             "spread": {"spread": True}, "pairs": {"pairs": True}}
    gsets = {f"gp_{k}": v for k, v in sets.items()}
    eng.candidate_refs_upload(beam_refs(C))
    kinds.update({k: {"groups": True} for k in sets})
    kinds.update({k: {"group_pairs": True} for k in gsets})
    last, times, med = timed(eng, C, K, steps, score_kw, kinds, {**sets, **gsets})
    ok = [same(last["candidates"].candidates[c], d) for c, d in zip(picks, ref)]
    import exact_report as xr
    cc = last["candidate_corpus"].candidate_corpus
    exact = [[list(x) for x in xr.diff_exact(cc[c], d)] for c, d in zip(picks, ref_corpus["exact"])]
    seq = [seq_corpus_diff(cc[c], d) for c, d in zip(picks, ref_corpus["seq"])]
    return {**groups_block(last, med, sets, None), "groups_bytes": b"".join(bytes(last[k].groups) for k in sets),
            **spread_block(eng, last, med, None), "spread_bytes": bytes(last["spread"].spread),
            **pairs_block(last, med, None), "pairs_bytes": bytes(last["pairs"].pairs),
            **group_pairs_block(last, med, gsets, None), "group_pairs_bytes": b"".join(bytes(last[k].group_pairs) for k in gsets),
            "plain_ms_median": round(med["plain"], 3), "candidates_ms_median": round(med["candidates"], 3),
            "candidate_corpus_ms_median": round(med["candidate_corpus"], 3),
            "candidates_ratio": round(med["candidates"] / med["plain"], 3),
            "candidate_corpus_ratio": round(med["candidate_corpus"] / med["plain"], 3),
            "extremes_ms_median": round(med["extremes"], 3), "extremes_ratio": round(med["extremes"] / med["plain"], 3),
            "parity_extremes": extremes_parity(last["extremes"], None), "extremes_bytes": bytes(last["extremes"].extremes),
            "min_ms": {k: round(min(v) * 1e3, 3) for k, v in times.items()},
            "parity": {"candidates": picks, "equal": all(ok), "per_candidate": ok},
            "parity_corpus": {**parity_block(picks, exact), "check": "exact report, every field bit for bit",
                              "pattern_counts": [[int(cc[c].pat[p].count) for p in range(6)] for c in picks]},
            "parity_corpus_seq": {**parity_block(picks, seq), "check": "oracle.report, binary64 sums to 1e-12"}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out")
    ap.add_argument("--legs", default="D,Q,T,R16")
    args = ap.parse_args()
    import importlib
    pkg = importlib.import_module("senweaver-ide_b200")
    import oracle
    from oracle import candidates as oc
    import exact_report as xr
    import extremes_fixtures as xf
    import group_fixtures as gf
    import spread_fixtures as sf
    import pair_fixtures as pf
    import group_pair_fixtures as gpf
    legs = args.legs.split(",")
    out = {"card": card(), "steps": args.steps, "timing": "host clock around each synchronous apo_score call"}
    eng = pkg.Engine(0)
    seed, C, T, K = 0x5EED0003, 256, 5_000_000, 4
    picks = [int(x) for x in np.linspace(0, C - 1, 8).round()]
    nth = max(1, min(32, os.cpu_count() or 1))
    try:
        if {"D", "W", "Q", "T"} & set(legs):
            ref = oc.cand_generated(seed, picks, 0, T, 300, nthreads=nth)
            sets = label_sets(T)
            ref_ext, ref_grp, ref_spr = {}, {}, {}
            for c in (picks[0], picks[-1]):
                d = oracle.gen_dims(seed, c, 1, 0, T, 300, nth)
                ref_ext[c] = xf.model(d)[0]
                ref_grp[c] = {k: gf.model(d, lab, G)[0] for k, (lab, G) in sets.items()}
                ref_spr[c] = sf.model(d)[0]
                del d
            refs, ref_pair, ref_gpair = beam_refs(C), {}, {}
            for c in (1, C - 2):                            # a child of candidate 0 and one of the last block's
                r = int(refs[c])
                d = np.concatenate([oracle.gen_dims(seed, c, 1, 0, T, 300, nth), oracle.gen_dims(seed, r, 1, 0, T, 300, nth)])
                ref_pair[c] = pf.model(d, [1, pf.NONE])[0] | {"ref": r}
                ref_gpair[c] = {k: [m | {"ref": r} for m in gpf.model(d, [1, pf.NONE], lab, G)[0]] for k, (lab, G) in sets.items()}
                del d
            if "D" in legs:
                eng.dims_generate(seed, 0, C, 0, T, 300)
                out["form_d_256x5M"] = leg(eng, C, K, args.steps, {}, ref, picks, ref_ext, sets, ref_grp, ref_spr, ref_pair, ref_gpair)
            if "W" in legs:
                eng.dims_generate(seed, 0, C, 0, T, 300)
                eng.set_tuning(pkg.TUNE_NO_TWIN_T)
                out["form_w_copy_256x5M"] = leg(eng, C, K, args.steps, {}, ref, picks, ref_ext, sets, ref_grp, ref_spr, ref_pair, ref_gpair)
                eng.set_tuning(0)
            if "Q" in legs or "T" in legs:
                eng.dims_generate_compact(seed, 0, C, 0, T, 300)
            if "Q" in legs:
                out["form_q_256x5M"] = leg(eng, C, K, args.steps, {}, ref, picks, ref_ext, sets, ref_grp, ref_spr, ref_pair, ref_gpair)
            if "T" in legs:
                pc, pd = np.empty((C, T), np.uint32), np.empty((C, T), np.uint16)
                for c in range(C):
                    eng.dims_packed_download(c, 0, T, out=(pc[c], pd[c]))
                book, d2book = eng.dims_codebook(), eng.dims_d2book()
                tl, th, tbook = pkg.tuple_encode_host(pc, pd, nthreads=nth)
                del pc, pd
                eng.tuples_upload(tl, th, tbook, book, d2book)
                del tl, th
                out["form_t_256x5M"] = leg(eng, C, K, args.steps, {"source": pkg.SRC_TUPLES}, ref, picks, ref_ext, sets, ref_grp, ref_spr, ref_pair, ref_gpair)
        if {"R16", "R"} & set(legs):
            Cr = 128
            picks_r = [int(x) for x in np.linspace(0, Cr - 1, 8).round()]
            ref_r = oc.cand_generated(seed, picks_r, 0, T, 300, nthreads=nth, records=True)
            ref_rc = {"seq": [oracle.report(oracle.gen_records(seed, oracle.STREAM_ROLLOUT, c, 1, 0, T, 300, nth), nthreads=nth)
                              for c in picks_r]}
            ref_rc["exact"] = [xr.combine(q, d) for q, d in zip(ref_rc["seq"], ref_r)]
            if "R16" in legs:
                eng.rollouts16_generate(seed, 0, Cr, 0, T, 300)
                out["form_r16_128x5M"] = corpus_leg(eng, Cr, K, args.steps, {"source": pkg.SRC_ROLLOUTS}, ref_r, picks_r, ref_rc, label_sets(T))
            if "R" in legs:
                eng.rollouts_generate(seed, 0, Cr, 0, T, 300)
                out["form_r_128x5M"] = corpus_leg(eng, Cr, K, args.steps, {"source": pkg.SRC_ROLLOUTS}, ref_r, picks_r, ref_rc, label_sets(T))
            if "R16" in legs and "R" in legs:                   # the same rollouts: the same lists
                out["r16_r_extremes_equal"] = out["form_r16_128x5M"]["extremes_bytes"] == out["form_r_128x5M"]["extremes_bytes"]
                out["r16_r_groups_equal"] = out["form_r16_128x5M"]["groups_bytes"] == out["form_r_128x5M"]["groups_bytes"]
                out["r16_r_spread_equal"] = out["form_r16_128x5M"]["spread_bytes"] == out["form_r_128x5M"]["spread_bytes"]
                out["r16_r_pairs_equal"] = out["form_r16_128x5M"]["pairs_bytes"] == out["form_r_128x5M"]["pairs_bytes"]
                out["r16_r_group_pairs_equal"] = out["form_r16_128x5M"]["group_pairs_bytes"] == out["form_r_128x5M"]["group_pairs_bytes"]
            for k in ("form_r16_128x5M", "form_r_128x5M"):
                out.get(k, {}).pop("extremes_bytes", None)
                out.get(k, {}).pop("groups_bytes", None)
                out.get(k, {}).pop("spread_bytes", None)
                out.get(k, {}).pop("pairs_bytes", None)
                out.get(k, {}).pop("group_pairs_bytes", None)
        if "FALL" in legs:
            Cf, Tf = 64, 1_000_000
            d = xf.falling(Tf, 1)
            m = xf.model(d)[0]
            sets_f = label_sets(Tf)
            mg = {k: gf.model(d, lab, G)[0] for k, (lab, G) in sets_f.items()}
            eng.dims_upload(np.repeat(d, Cf, axis=0))
            eng.set_tuning(pkg.TUNE_NO_TWIN)
            out["falling_rows_k1_64x1M"] = leg(eng, Cf, K, args.steps, {}, None, None, {0: m, Cf - 1: m}, sets_f, {0: mg, Cf - 1: mg},
                                               {0: sf.model(d)[0], Cf - 1: sf.model(d)[0]},
                                               {c: pf.model(np.concatenate([d, d]), [1, pf.NONE])[0] | {"ref": int(beam_refs(Cf)[c])}
                                                for c in (1, Cf - 2)})
            eng.set_tuning(0)
    finally:
        eng.close()
    out["card_after"] = card()
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
