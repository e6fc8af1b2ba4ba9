"""What reading the Form T copy from its 16-bit plane buys (K1t2, 2 B per evaluation plus the exception list) against
reading both planes (K1t, 3 B per evaluation), and the sweep behind the list's eligibility bound (at most 1/64 of the
evaluations as exceptions).

  flagship   the configs[2] step (256 x 5 M Form D + the 5 M-record corpus, one apo_score call) on one engine, alternating
             blocks with TUNE_NO_TWIN_T2 set (K1t) and clear (K1t2); apo_dims_generate's wall time with and without the
             list; the exception share and the bytes each route reads per evaluation; identical integers, scores, counts,
             top-K and report; one torch.profiler record of a K1t2 step.
  sweep      K1t2 against K1t over 64 x 1 M evaluations with 1/1024, 1/256, 1/128 and 1/64 of them exceptions (65 536
             frequent evaluations and rare ones seen once, as tests/test_gpu_twin_t_list.py builds them), a fresh
             engine for each.

    python examples/form_d_tuple_copy16.py [--steps 20] [--rounds 3] [--skip-flagship] [--skip-sweep] [--out FILE.json]

Prints one JSON object; the card name and power limit are read in the same run (nvidia-smi query)."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
from form_d_tuple_copy import profile_step, stats, timed  # noqa: E402
from form_d_twin import card  # noqa: E402
from test_gpu_dims_tuple_copy import kernels  # noqa: E402


def kernel_of(names):
    return "K1t2" if "k_reward9t2" in names else "K1t" if "k_reward9t" in names else "other"


def share(eng, N):
    got = eng.debug_twin_t_list()
    return 0 if got is None else len(got[1]), N


def ab(eng, pkg, call, C, N, torch, stream, steps, rounds, warmup, corpus_T=0):
    """alternating blocks of the two routes on one engine: step and kernel times, bytes, identical results"""
    settings = {"t3": pkg.TUNE_NO_TWIN_T2, "t2": 0}
    step = {n: [] for n in settings}
    kern = {n: [] for n in settings}
    last = {}
    for _ in range(rounds):
        for name, flags in settings.items():
            eng.set_tuning(flags)
            s, k, r = timed(torch, eng, stream, call, steps, warmup)
            step[name] += s
            kern[name] += k
            last[name] = (r, eng.debug_partials(C))
    n_ex, _ = share(eng, N)
    out = {"exceptions": n_ex, "exception_share": round(n_ex / N, 6)}
    for name, flags in settings.items():
        eng.set_tuning(flags)
        held = kernel_of(kernels(call))
        per_eval = 3.0 if held == "K1t" else 2.0 + 8.0 * n_ex / N        # the list: {position, index} per exception
        moved = per_eval * N + 32 * corpus_T
        out[name] = {"kernel": held, "ms_per_step": stats(step[name]), "kernel_ms": stats(kern[name]),
                     "bytes_per_eval": round(per_eval, 4), "kernel_GBps": round(moved / (float(np.median(kern[name])) * 1e-3) / 1e9, 1)}
    eng.set_tuning(0)
    (ra, pa), (rb, pb) = last["t3"], last["t2"]
    out["identical"] = {"integers": pa == pb, "scores": bool(np.array_equal(ra.scores, rb.scores)),
                        "counts": bool(np.array_equal(ra.counts, rb.counts)), "topk": bool(np.array_equal(ra.topk, rb.topk))}
    if ra.report is not None:
        out["identical"]["report_bad"] = ra.report.bad == rb.report.bad
    out["step_speedup"] = round(out["t3"]["ms_per_step"]["median"] / out["t2"]["ms_per_step"]["median"], 3)
    out["kernel_speedup"] = round(out["t3"]["kernel_ms"]["median"] / out["t2"]["kernel_ms"]["median"], 3)
    return out


def flagship(eng, pkg, torch, stream, steps, rounds, warmup):
    seed, C, T, K = 0x5EED0003, 256, 5_000_000, 64
    load = {"no_list": [], "list": []}
    for _ in range(3):
        for name, flags in (("no_list", pkg.TUNE_NO_TWIN_T2), ("list", 0)):
            eng.set_tuning(flags)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eng.dims_generate(seed, 0, C, 0, T, 300)                       # synchronous; the last one holds the list
            load[name].append(time.perf_counter() - t0)
    eng.corpus_generate(seed, 0, T, 300)
    call = lambda: eng.score(C, K, corpus=True)
    out = {"workload": f"{C} x {T} Form D + {T}-record corpus, apo_score with the corpus report, K={K}",
           "dims_generate_s": {n: stats(v) for n, v in load.items()}}
    out.update(ab(eng, pkg, call, C, C * T, torch, stream, steps, rounds, warmup, corpus_T=T))
    out["launches"] = call().timing.launches
    out["profile"] = profile_step(torch, call)
    return out


def sweep(pkg, torch, stream, steps, rounds, warmup):
    import test_gpu_twin_t_list as t
    C, T = 64, 1 << 20
    rng = np.random.default_rng(11)
    out = {}
    for inv in (1024, 256, 128, 64):
        rare = np.zeros((C, T), bool)
        rare.reshape(-1)[rng.choice(C * T, C * T // inv, replace=False)] = True
        dims = t.tensor(12 + inv, C, T, rare)
        eng = pkg.Engine(0)
        try:
            eng.set_stream(stream.cuda_stream)
            eng.dims_upload(dims)                                          # 2^26 evaluations: the copy by the size rule
            del dims
            out[f"1/{inv}"] = ab(eng, pkg, lambda: eng.score(C, 4), C, C * T, torch, stream, steps, rounds, warmup)
        finally:
            eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--skip-flagship", action="store_true")
    ap.add_argument("--skip-sweep", action="store_true")
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    pkg = importlib.import_module("senweaver-ide_b200")
    out = {"card": card(), "timing": "CUDA events around each apo_score call on the engine's stream; kernel time from apo_last_timing"}
    stream = torch.cuda.current_stream()
    ok = True
    if not args.skip_flagship:
        eng = pkg.Engine(0)
        eng.set_stream(stream.cuda_stream)
        try:
            out["flagship"] = flagship(eng, pkg, torch, stream, args.steps, args.rounds, args.warmup)
            ok &= all(out["flagship"]["identical"].values())
        finally:
            eng.close()
    if not args.skip_sweep:
        out["sweep"] = sweep(pkg, torch, stream, args.steps, args.rounds, args.warmup)
        ok &= all(all(v["identical"].values()) for v in out["sweep"].values())
    out["card_after"] = card()
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
