"""What the per-candidate breakdown (APO_SCORE_CANDIDATES) costs: the flagged scoring step beside the plain one, in the
same process, alternating, on the configs[2] workload (256 x 5 M) resident as Form D, Form Q and Form T, and on 128 x 5 M
Form R16 rollouts.  Every leg carries a parity block: the full breakdown of 8 candidates spread over C, over the whole
record axis, against the CPU oracle's generator path (integers, first-three examples and every binary64 field).

    python examples/candidates_cost.py [--steps 10] [--out FILE.json]

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


def leg(eng, C, K, steps, score_kw, ref, picks):
    plain, flagged = [], []
    for _ in range(2):                                          # warm both shapes
        eng.score(C, K, **score_kw)
        eng.score(C, K, candidates=True, **score_kw)
    for _ in range(steps):                                      # alternate: drift and other tenants hit both alike
        t0 = time.perf_counter(); eng.score(C, K, **score_kw); plain.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); r = eng.score(C, K, candidates=True, **score_kw); flagged.append(time.perf_counter() - t0)
    ok = [same(r.candidates[c], d) for c, d in zip(picks, ref)]
    med_p, med_f = float(np.median(plain)) * 1e3, float(np.median(flagged)) * 1e3
    return {"plain_ms_median": round(med_p, 3), "flagged_ms_median": round(med_f, 3), "ratio": round(med_f / med_p, 3),
            "plain_ms_min": round(min(plain) * 1e3, 3), "flagged_ms_min": round(min(flagged) * 1e3, 3),
            "parity": {"candidates": picks, "equal": all(ok), "per_candidate": ok,
                       "bad_examples": [list(r.candidates[c].badExamples) for c in picks]}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out")
    ap.add_argument("--legs", default="D,Q,T,R16")
    args = ap.parse_args()
    import importlib
    pkg = importlib.import_module("senweaver-ide_b200")
    from oracle import candidates as oc
    legs = args.legs.split(",")
    out = {"card": card(), "steps": args.steps, "timing": "host clock around each synchronous apo_score call"}
    eng = pkg.Engine(0)
    seed, C, T, K = 0x5EED0003, 256, 5_000_000, 4
    picks = [int(x) for x in np.linspace(0, C - 1, 8).round()]
    nth = max(1, min(32, os.cpu_count() or 1))
    try:
        if {"D", "Q", "T"} & set(legs):
            ref = oc.cand_generated(seed, picks, 0, T, 300, nthreads=nth)
            if "D" in legs:
                eng.dims_generate(seed, 0, C, 0, T, 300)
                out["form_d_256x5M"] = leg(eng, C, K, args.steps, {}, ref, picks)
            if "Q" in legs or "T" in legs:
                eng.dims_generate_compact(seed, 0, C, 0, T, 300)
            if "Q" in legs:
                out["form_q_256x5M"] = leg(eng, C, K, args.steps, {}, ref, picks)
            if "T" in legs:
                pc, pd = np.empty((C, T), np.uint32), np.empty((C, T), np.uint16)
                for c in range(C):
                    eng.dims_packed_download(c, 0, T, out=(pc[c], pd[c]))
                book, d2book = eng.dims_codebook(), eng.dims_d2book()
                tl, th, tbook = pkg.tuple_encode_host(pc, pd, nthreads=nth)
                del pc, pd
                eng.tuples_upload(tl, th, tbook, book, d2book)
                del tl, th
                out["form_t_256x5M"] = leg(eng, C, K, args.steps, {"source": pkg.SRC_TUPLES}, ref, picks)
        if "R16" in legs:
            Cr = 128
            picks_r = [int(x) for x in np.linspace(0, Cr - 1, 8).round()]
            ref_r = oc.cand_generated(seed, picks_r, 0, T, 300, nthreads=nth, records=True)
            eng.rollouts16_generate(seed, 0, Cr, 0, T, 300)
            out["form_r16_128x5M"] = leg(eng, Cr, K, args.steps, {"source": pkg.SRC_ROLLOUTS}, ref_r, picks_r)
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
