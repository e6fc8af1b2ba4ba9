"""What the compact copy of a resident Form D tensor buys: the configs[2] step (256 x 5 M Form D + the 5 M-record corpus, one
apo_score call) on one engine, alternating blocks with TUNE_NO_TWIN set (K1 reads the 36 B/eval fp32 tensor) and clear (K1q
reads the copy built at load: Form W words, 8 B/eval, when no coded dimension has more than 15 values, else the 14 B/eval
Form Q planes).  Reports which copy is held (from the K1q instantiation a profiler record shows), per setting the ms/step
median and spread, the scoring kernel's time and the bytes it moved per second (36, 14 or 8 B per evaluation + 32 B per corpus
record), whether the two settings gave identical integers, scores and top-K, and the wall time of apo_dims_generate with and
without building the copy.

    python examples/form_d_twin.py [--steps 20] [--rounds 3] [--out FILE.json]

Prints one JSON object; the card name and power limit are read in the same run (nvidia-smi query)."""
import argparse
import importlib
import json
import os
import re
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


def held_copy(fn):
    """'W' or 'Q': the layout the K1q launch of fn() read (last template argument of k_reward9q), None if K1q did not run"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    for ev in prof.events():
        m = re.search(r"k_reward9q<([^>]*)>", ev.name)
        if m:
            return "W" if m.group(1).split(",")[-1].strip() == "true" else "Q"
        m = re.search(r"k_reward9qI(.*)EEvNS_8KqParams", ev.name)       # not demangled
        if m:
            return "W" if m.group(1).endswith("Lb1EE") else "Q"
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="timed steps per block")
    ap.add_argument("--rounds", type=int, default=3, help="blocks per setting, alternating")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    pkg = importlib.import_module("senweaver-ide_b200")
    seed, C, T, K = 0x5EED0003, 256, 5_000_000, 64
    settings = {"k1_fp32": pkg.TUNE_NO_TWIN, "k1q_copy": 0}
    out = {"card": card(), "workload": f"{C} x {T} Form D + {T}-record corpus, apo_score with the corpus report, K={K}",
           "timing": "CUDA events around each apo_score call on the engine's stream; kernel time from apo_last_timing"}
    eng = pkg.Engine(0)
    try:
        # load cost: apo_dims_generate without (TUNE_NO_TWIN) and with building the copy, alternating
        load = {name: [] for name in settings}
        for _ in range(3):
            for name, flags in settings.items():
                eng.set_tuning(flags)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                eng.dims_generate(seed, 0, C, 0, T, 300)                # synchronous
                load[name].append(time.perf_counter() - t0)
        out["dims_generate_s"] = {name: {"median": round(float(np.median(v)), 4), "min": round(min(v), 4), "max": round(max(v), 4)}
                                  for name, v in load.items()}
        # the last load (flags 0) holds the copy; TUNE_NO_TWIN from here on only stops it being read
        eng.corpus_generate(seed, 0, T, 300)
        copy = held_copy(lambda: eng.score(C, K, corpus=True))
        out["copy"] = {"W": "Form W (8 B/eval)", "Q": "Form Q (14 B/eval)"}.get(copy, "none")
        stream = torch.cuda.current_stream()
        eng.set_stream(stream.cuda_stream)
        steps = {name: [] for name in settings}
        kernel = {name: [] for name in settings}
        last = {}
        for _ in range(args.rounds):
            for name, flags in settings.items():
                eng.set_tuning(flags)
                for _ in range(args.warmup):
                    eng.score(C, K, corpus=True)
                for _ in range(args.steps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(stream)
                    r = eng.score(C, K, corpus=True)
                    e1.record(stream)
                    e1.synchronize()
                    steps[name].append(e0.elapsed_time(e1))
                    kernel[name].append(r.timing.reward_ms)
                last[name] = (r, eng.debug_partials(C))
        eng.set_tuning(0)
        eng.set_stream(0)
        per_eval = {"k1_fp32": 36, "k1q_copy": 8 if copy == "W" else 14}
        for name in settings:
            s, k = np.array(steps[name]), np.array(kernel[name])
            moved = per_eval[name] * C * T + 32 * T
            out[name] = {"ms_per_step_median": round(float(np.median(s)), 3), "ms_per_step_min": round(float(s.min()), 3),
                         "ms_per_step_max": round(float(s.max()), 3), "spread": round(float((s.max() - s.min()) / np.median(s)), 4),
                         "kernel_ms_median": round(float(np.median(k)), 3), "bytes_per_eval": per_eval[name],
                         "bytes_moved_per_step": moved, "kernel_GBps": round(moved / (float(np.median(k)) * 1e-3) / 1e9, 1),
                         "steps": int(s.size)}
        (ra, pa), (rb, pb) = last["k1_fp32"], last["k1q_copy"]
        out["identical"] = {"integers": pa == pb, "scores": bool(np.array_equal(ra.scores, rb.scores)),
                            "counts": bool(np.array_equal(ra.counts, rb.counts)), "topk": bool(np.array_equal(ra.topk, rb.topk)),
                            "report_bad": ra.report.bad == rb.report.bad}
        out["speedup_median"] = round(out["k1_fp32"]["ms_per_step_median"] / out["k1q_copy"]["ms_per_step_median"], 3)
    finally:
        eng.close()
    out["card_after"] = card()
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    sys.exit(0 if all(out.get("identical", {"ok": False}).values()) else 1)


if __name__ == "__main__":
    main()
