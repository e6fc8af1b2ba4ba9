"""What scoring whole rows of the Form T copy from its per-row dictionary counts buys (K1h, 8 B per distinct (row, entry)
pair) against reading its 16-bit slot plane (K1t2, 2 B per evaluation plus the lists).

The flagship step (256 x 5 M Form D + the 5 M-record corpus, one apo_score call with the corpus report) on one engine,
alternating blocks with TUNE_NO_TWIN_H clear (K1h) and set after the load (K1t2): step and K1 time of both routes, the
number of pairs, the bytes each route reads per evaluation and K1h's rate over its own bytes; apo_dims_generate's wall
time with and without the counts (medians of 3); identical integers, scores, counts, top-K and report.  The card's name,
power limit and max SM clock are read in the same run.

    python examples/form_d_counts.py [--steps 60] [--rounds 3] [--warmup 5] [--out FILE.json]

Prints one JSON object.  roofline figures elsewhere in the project still count 36 B per evaluation (the Form D tensor)."""
import argparse
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "examples"))
from form_d_tuple_copy import profile_step, stats, timed  # noqa: E402
from form_d_twin import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    pkg = importlib.import_module("senweaver-ide_b200")
    seed, C, T, K = 0x5EED0003, 256, 5_000_000, 64
    N = C * T
    out = {"card": card(), "workload": f"{C} x {T} Form D + {T}-record corpus, apo_score with the corpus report, K={K}",
           "timing": "CUDA events around each apo_score call on the engine's stream; K1 time from apo_last_timing"}
    stream = torch.cuda.current_stream()
    eng = pkg.Engine(0)
    eng.set_stream(stream.cuda_stream)
    ok = True
    try:
        load = {"no_counts": [], "counts": []}
        for _ in range(3):
            for name, flags in (("no_counts", pkg.TUNE_NO_TWIN_H), ("counts", 0)):
                eng.set_tuning(flags)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                eng.dims_generate(seed, 0, C, 0, T, 300)                        # synchronous; the last one holds the counts
                load[name].append(time.perf_counter() - t0)
        out["dims_generate_s"] = {n: stats(v) for n, v in load.items()}
        eng.set_tuning(0)
        got = eng.debug_twin_h()
        nnz = 0 if got is None else len(got[1])
        xl = eng.debug_twin_t_list()
        n_listed = 0 if xl is None else len(xl[1])
        out["pairs"] = nnz
        eng.corpus_generate(seed, 0, T, 300)
        call = lambda: eng.score(C, K, corpus=True)
        settings = {"k1h": 0, "k1t2": pkg.TUNE_NO_TWIN_H}
        per_eval = {"k1h": 8.0 * nnz / N, "k1t2": 2.0 + 8.0 * n_listed / N}
        step = {n: [] for n in settings}
        kern = {n: [] for n in settings}
        last = {}
        for _ in range(args.rounds):
            for name, flags in settings.items():
                eng.set_tuning(flags)
                s, k, r = timed(torch, eng, stream, call, args.steps, args.warmup)
                step[name] += s
                kern[name] += k
                last[name] = (r, eng.debug_partials(C))
        for name in settings:
            km = float(np.median(kern[name]))
            out[name] = {"ms_per_step": stats(step[name]), "k1_ms": stats(kern[name]), "bytes_per_eval": round(per_eval[name], 4),
                         "k1_GBps_own_bytes": round(per_eval[name] * N / (km * 1e-3) / 1e9, 1)}
        (ra, pa), (rb, pb) = last["k1h"], last["k1t2"]
        out["identical"] = {"integers": pa == pb, "scores": bool(np.array_equal(ra.scores, rb.scores)),
                            "counts": bool(np.array_equal(ra.counts, rb.counts)), "topk": bool(np.array_equal(ra.topk, rb.topk)),
                            "report": memoryview(ra.report).tobytes() == memoryview(rb.report).tobytes()}
        ok = all(out["identical"].values()) and nnz > 0
        out["step_speedup"] = round(out["k1t2"]["ms_per_step"]["median"] / out["k1h"]["ms_per_step"]["median"], 3)
        out["k1_speedup"] = round(out["k1t2"]["k1_ms"]["median"] / out["k1h"]["k1_ms"]["median"], 3)
        eng.set_tuning(0)
        out["launches"] = call().timing.launches
        out["profile"] = profile_step(torch, call)
    finally:
        eng.close()
    out["card_after"] = card()
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
