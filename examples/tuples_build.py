"""What building resident Form T on the device costs and buys (apo_dims_tuples).  Per workload (C x T Form D generated on the
device with bench.py's generator and seed, its Form W copy held, plus a T-record corpus):

  - the device build: median and spread of repeated synchronous apo_dims_tuples calls on one engine (host clock around each),
    and the kernel times of one profiled build (torch.profiler, a separate call) against the bytes the two passes must move;
  - the flagship step (apo_score with the corpus report) on SRC_TUPLES and on SRC_DIMS (which reads the Form W copy),
    alternating blocks in one run, CUDA events around each call, and whether both gave the same integers, scores and top-K;
  - n_tuples, and the number of steps after which the build has paid for itself;
  - the host route for comparison (apo_dims_download of every row + apo_packed_encode_host + apo_tuple_encode_host +
    apo_tuples_upload) where host memory holds the fp32 tensor, and whether it gave the same bytes.

    python examples/tuples_build.py [--shapes 256x5000000,64x1000000] [--builds 5] [--steps 20] [--rounds 3] [--out FILE.json]

Prints one JSON object; the card name and power limit are read in the same run (nvidia-smi query)."""
import argparse
import hashlib
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SEED = 0x5EED0003                 # bench.py's seed
HBM_BPS = 3.35e12                 # H100 SXM data sheet


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:
        return f"unknown ({ex})"


def stats(v):
    v = np.asarray(v, float)
    return {"median": round(float(np.median(v)), 3), "min": round(float(v.min()), 3), "max": round(float(v.max()), 3), "n": int(v.size)}


def digest(eng, C, T):
    h = hashlib.sha256()
    (pc, pd), cb, d2 = eng.tuples_book()
    for a in (pc, pd, cb, d2):
        h.update(a.tobytes())
    for c in range(C):
        for a in eng.tuples_download(c, 0, T):
            h.update(a.tobytes())
    return h.hexdigest()


def host_available():
    try:
        with open("/proc/meminfo") as f:
            for line in f:
                if line.startswith("MemAvailable:"):
                    return int(line.split()[1]) * 1024
    except OSError:
        pass
    return 0


def kernel_ms(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.events():
        for k in ("k_tb_count", "k_tb_index", "k_tb_clear", "k_tb_compact", "k_tb_insert"):
            if k in ev.name:
                out[k] = round(out.get(k, 0.0) + ev.device_time_total / 1e3, 3)
    return out


def workload(pkg, C, T, args):
    import torch
    out = {"workload": f"{C} x {T} Form D (apo_dims_generate, seed {SEED:#x}) + {T}-record corpus, K=64"}
    eng = pkg.Engine(0)
    try:
        eng.dims_generate(SEED, 0, C, 0, T, 300)
        eng.corpus_generate(SEED, 0, T, 300)
        n = eng.dims_tuples()                                           # warm-up (module load, first allocations)
        builds = []
        for _ in range(args.builds):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            n = eng.dims_tuples()                                       # synchronous
            builds.append((time.perf_counter() - t0) * 1e3)
        out["n_tuples"] = n
        out["build_ms"] = stats(builds)
        ks = kernel_ms(eng.dims_tuples)
        src_bytes = C * T * 8                                           # Form W words, read by both passes
        moved = 2 * src_bytes + C * T * 3
        out["build_kernels_ms"] = ks
        out["build_bytes_moved"] = moved
        out["build_bound_ms_at_datasheet_hbm"] = round(moved / HBM_BPS * 1e3, 3)
        if "k_tb_count" in ks and "k_tb_index" in ks:
            out["count_pass_GBps"] = round(src_bytes / (ks["k_tb_count"] * 1e-3) / 1e9, 1)
            out["index_pass_GBps"] = round((src_bytes + C * T * 3) / (ks["k_tb_index"] * 1e-3) / 1e9, 1)
        # the step, alternating sources
        stream = torch.cuda.current_stream()
        eng.set_stream(stream.cuda_stream)
        srcs = {"tuples": pkg.SRC_TUPLES, "dims_w_copy": pkg.SRC_DIMS}
        steps = {k: [] for k in srcs}
        last = {}
        for _ in range(args.rounds):
            for name, src in srcs.items():
                for _ in range(args.warmup):
                    eng.score(C, 64, source=src, corpus=True)
                for _ in range(args.steps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(stream)
                    r = eng.score(C, 64, source=src, corpus=True)
                    e1.record(stream)
                    e1.synchronize()
                    steps[name].append(e0.elapsed_time(e1))
                last[name] = (r, eng.debug_partials(C))
        eng.set_stream(0)
        for name in srcs:
            out[f"step_ms_{name}"] = stats(steps[name])
        (ra, pa), (rb, pb) = last["tuples"], last["dims_w_copy"]
        out["identical"] = {"integers": pa == pb, "scores": ra.scores.tobytes() == rb.scores.tobytes(), "topk": bool(np.array_equal(ra.topk, rb.topk)),
                            "report": bytes(ra.report) == bytes(rb.report)}
        gain = out["step_ms_dims_w_copy"]["median"] - out["step_ms_tuples"]["median"]
        out["steps_to_pay_for_build"] = round(out["build_ms"]["median"] / gain, 2) if gain > 0 else None
        # the host route
        need = C * T * (36 + 6 + 3) + (1 << 30)
        if args.host_route and host_available() > need:
            dev = digest(eng, C, T)
            t0 = time.perf_counter()
            dims = np.empty((C, T, 9), np.float32)
            for c in range(C):
                dims[c] = eng.dims_download(c, 0, T)
            t1 = time.perf_counter()
            pc, pd, book, d2book = pkg.packed_encode_host(dims, nthreads=os.cpu_count() or 8)
            t2 = time.perf_counter()
            del dims
            tl, th, tb = pkg.tuple_encode_host(pc, pd, nthreads=os.cpu_count() or 8)
            t3 = time.perf_counter()
            eng.tuples_upload(tl, th, tb, book, d2book)
            t4 = time.perf_counter()
            out["host_route_s"] = {"dims_download": round(t1 - t0, 3), "packed_encode_host": round(t2 - t1, 3),
                                   "tuple_encode_host": round(t3 - t2, 3), "tuples_upload": round(t4 - t3, 3), "total": round(t4 - t0, 3),
                                   "host_threads": os.cpu_count()}
            out["host_route_same_bytes"] = digest(eng, C, T) == dev
        else:
            out["host_route_s"] = f"not measured: host memory available {host_available() >> 30} GiB, needs {need >> 30} GiB" \
                if args.host_route else "not measured (--no-host-route)"
    finally:
        eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="256x5000000,64x1000000")
    ap.add_argument("--builds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-host-route", dest="host_route", action="store_false")
    ap.add_argument("--out")
    args = ap.parse_args()
    pkg = importlib.import_module("senweaver-ide_b200")
    res = {"card": card(), "timing": "build: host clock around synchronous apo_dims_tuples calls; step: CUDA events around apo_score",
           "workloads": []}
    for s in args.shapes.split(","):
        C, T = (int(x) for x in s.split("x"))
        res["workloads"].append(workload(pkg, C, T, args))
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    ok = all(all(w["identical"].values()) and w.get("host_route_same_bytes", True) for w in res["workloads"])
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
