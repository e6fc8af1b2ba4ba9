"""What the Form T copy of a resident Form D tensor buys, and where its size rule and dictionary cap come from.

  flagship   the configs[2] step (256 x 5 M Form D + the 5 M-record corpus, one apo_score call) on one engine, alternating
             blocks with TUNE_NO_TWIN_T set (K1q reads the 8 B/eval Form W copy) and clear (K1t reads the 3 B/eval Form T
             copy); apo_dims_generate's wall time with and without building the copy; identical integers, scores, counts,
             top-K and report; one torch.profiler record of a Form T step (kernels, durations, gaps).
  sizes      the same at 256 x 262 144 (2^26 = 67 M evaluations), 256 x 625 k (160 M) and 256 x 5 M: build cost, per-step saving,
             steps to pay the build back.
  dictionary K1t against K1q on Form W over 16 x 4 M evaluations drawn uniformly from 2^15, 2^18, 2^20 and 2^22 distinct
             ones (K1t through apo_dims_tuples + SRC_TUPLES: the same kernel the copy runs).

    python examples/form_d_tuple_copy.py [--steps 20] [--rounds 3] [--skip-sizes] [--skip-dictionary] [--out FILE.json]

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
from form_d_twin import card  # noqa: E402
from test_gpu_dims_twin import kernels  # noqa: E402


def kernel_of(names):
    return "K1t" if "k_reward9t" in names else "K1q" if "k_reward9q" in names else "K1"


def timed(torch, eng, stream, call, steps, warmup):
    for _ in range(warmup):
        call()
    ms, kern = [], []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        r = call()
        e1.record(stream)
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
        kern.append(r.timing.reward_ms)
    return ms, kern, r


def stats(v):
    v = np.asarray(v)
    return {"median": round(float(np.median(v)), 4), "min": round(float(v.min()), 4), "max": round(float(v.max()), 4)}


def profile_step(torch, call):
    """kernels of one call, in launch order, with their durations and the gaps between them (us)"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    evs = sorted((e for e in prof.events() if e.device_type.name == "CUDA"), key=lambda e: e.time_range.start)
    out, end = [], None
    for e in evs:
        out.append({"name": e.name[:60], "us": round(e.time_range.end - e.time_range.start, 1),
                    "gap_us": None if end is None else round(e.time_range.start - end, 1)})
        end = e.time_range.end
    return out


def compare(eng, pkg, C, K, T, seed, steps, rounds, warmup, torch, stream, loads=3):
    settings = {"w_copy": pkg.TUNE_NO_TWIN_T, "t_copy": 0}
    load = {name: [] for name in settings}
    for _ in range(loads):
        for name, flags in settings.items():
            eng.set_tuning(flags)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eng.dims_generate(seed, 0, C, 0, T, 300)                       # synchronous; the last one (flags 0) holds the copy
            load[name].append(time.perf_counter() - t0)
    eng.corpus_generate(seed, 0, T, 300)
    call = lambda: eng.score(C, K, corpus=True)
    out = {"dims_generate_s": {n: stats(v) for n, v in load.items()}}
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
    for name, flags in settings.items():
        eng.set_tuning(flags)
        held = kernel_of(kernels(call))
        per_eval = 3 if held == "K1t" else 8
        moved = per_eval * C * T + 32 * T
        out[name] = {"kernel": held, "ms_per_step": stats(step[name]), "kernel_ms": stats(kern[name]), "bytes_per_eval": per_eval,
                     "kernel_bytes_per_step": moved, "kernel_GBps": round(moved / (float(np.median(kern[name])) * 1e-3) / 1e9, 1)}
    eng.set_tuning(0)
    (ra, pa), (rb, pb) = last["w_copy"], last["t_copy"]
    out["identical"] = {"integers": pa == pb, "scores": bool(np.array_equal(ra.scores, rb.scores)),
                        "counts": bool(np.array_equal(ra.counts, rb.counts)), "topk": bool(np.array_equal(ra.topk, rb.topk)),
                        "report_bad": ra.report.bad == rb.report.bad}
    saving = out["w_copy"]["ms_per_step"]["median"] - out["t_copy"]["ms_per_step"]["median"]
    build = out["dims_generate_s"]["t_copy"]["median"] - out["dims_generate_s"]["w_copy"]["median"]
    out["build_extra_s"] = round(build, 4)
    out["saving_ms_per_step"] = round(saving, 4)
    out["payback_steps"] = round(build * 1e3 / saving, 1) if saving > 0 else None
    out["speedup"] = round(out["w_copy"]["ms_per_step"]["median"] / out["t_copy"]["ms_per_step"]["median"], 3)
    return out, call


def dictionary_sweep(eng, pkg, torch, stream, steps, warmup):
    rng = np.random.default_rng(7)
    C, T = 16, 4 << 20
    levels = np.array([-1.0, -0.8, -0.5, -0.3, -0.2, 0.0, 0.3, 0.5, 0.8, 1.0], np.float32)
    d2 = rng.uniform(0, 1, 300).astype(np.float32)
    out = {}
    for bits in (15, 18, 20, 22):
        n = 1 << bits
        pool = levels[rng.integers(0, 10, (int(n * 1.1) + 64, 9))]
        pool[:, 2] = d2[rng.integers(0, 300, pool.shape[0])]
        pool = np.unique(pool, axis=0)[:n]
        rng.shuffle(pool)
        dims = np.empty((C, T, 9), np.float32)
        for c in range(C):
            dims[c] = pool[rng.integers(0, pool.shape[0], T)]
        eng.set_tuning(pkg.TUNE_NO_TWIN_T)
        eng.dims_upload(dims)
        del dims
        nt = eng.dims_tuples()
        eng.set_tuning(0)
        _, kw, rw = timed(torch, eng, stream, lambda: eng.score(C, 4), steps, warmup)
        pw = eng.debug_partials(C)
        _, kt, rt = timed(torch, eng, stream, lambda: eng.score(C, 4, source=pkg.SRC_TUPLES), steps, warmup)
        out[f"2^{bits}"] = {"distinct": nt, "k1q_w_ms": stats(kw), "k1t_ms": stats(kt),
                            "k1t_over_k1q": round(float(np.median(kt)) / float(np.median(kw)), 3),
                            "identical": pw == eng.debug_partials(C) and bool(np.array_equal(rw.topk, rt.topk))}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--skip-sizes", action="store_true")
    ap.add_argument("--skip-dictionary", action="store_true")
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    pkg = importlib.import_module("senweaver-ide_b200")
    seed, C, T, K = 0x5EED0003, 256, 5_000_000, 64
    out = {"card": card(), "workload": f"{C} x {T} Form D + {T}-record corpus, apo_score with the corpus report, K={K}",
           "timing": "CUDA events around each apo_score call on the engine's stream; kernel time from apo_last_timing"}
    eng = pkg.Engine(0)
    stream = torch.cuda.current_stream()
    eng.set_stream(stream.cuda_stream)
    ok = True
    try:
        flag, call = compare(eng, pkg, C, K, T, seed, args.steps, args.rounds, args.warmup, torch, stream)
        out["flagship"] = flag
        ok &= all(flag["identical"].values())
        out["flagship_profile"] = profile_step(torch, call)
        if not args.skip_sizes:
            out["sizes"] = {}
            for Ts in (262_144, 625_000):
                s, _ = compare(eng, pkg, C, K, Ts, seed, args.steps, 1, args.warmup, torch, stream, loads=2)
                out["sizes"][f"{C}x{Ts}"] = s
                ok &= all(s["identical"].values())
        if not args.skip_dictionary:
            eng.close()
            eng = pkg.Engine(0)
            eng.set_stream(stream.cuda_stream)
            out["dictionary"] = dictionary_sweep(eng, pkg, torch, stream, args.steps, args.warmup)
            ok &= all(v["identical"] for v in out["dictionary"].values())
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
