"""Where the flagship launch's time goes: K1h's pair stream, the corpus digest pass, the ticket and the finalising tail.

The flagship step (256 x 5 M Form D + the 5 M-record corpus, seed 0x5EED0003, one apo_score call with the corpus report, K=64)
is one launch of K1h (k_reward9th).  Per library, in a process of its own, --steps calls after --warmup:
  step_ms       CUDA events around each apo_score call on the engine's stream
  k1_ms         apo_last_timing's kernel time (timing.reward_ms), the whole launch
  host_gap_ms   step - k1_ms: the host-side part of the step (wrapper, ctypes, launch, synchronise)
  tail_finalize_ms / tail_publish_ms   the finalising CTA's own timers (segmented sum + report + top-K; the copy out)
With a build compiled with -DAPO_K1H_DIAG (made here into a temporary directory unless --diag-lib names one) it also reads
the %globaltimer stamps of every CTA (apo_corpus.cuh kh_stamp), as microseconds after the earliest CTA entry: the last CTA's
entry, the end of the last pairs, the end of the last digest share, the last ticket, the start and end of finalize_block
and the end of the publish; and the launch time of the stream alone (APO_K1H_DIAG=1: the gather replaced by a constant).
--lib runs the plain part on another build of the library (e.g. an earlier commit's).

    python examples/flagship_launch.py [--steps 60] [--warmup 5] [--rounds 3] [--diag-lib SO] [--lib SO] [--out FILE]

Prints one JSON object with the card's name, power limit and max SM clock read in the same run."""
import argparse
import ctypes
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "examples"))
SEED, C, T, K = 0x5EED0003, 256, 5_000_000, 64
STAMPS = ["entry", "pairs", "digest", "ticket", "finalize_start", "finalize_end", "publish"]   # apo_corpus.cuh KH_ST_*
NSTAMP, MAX_CTAS = 8, 256


def build_diag(tmp):
    """the library with the phase stamps and the stream-only variant, compiled from this tree's sources into tmp"""
    src = os.path.join(ROOT, "senweaver-ide_b200", "csrc")
    pkg = os.path.join(tmp, "pkg")
    shutil.copytree(src, os.path.join(pkg, "csrc"), ignore=shutil.ignore_patterns("*.o"))
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(tmp, "include"))
    r = subprocess.run(["make", "-s", "-C", os.path.join(pkg, "csrc"), "NVCC=nvcc -DAPO_K1H_DIAG"], capture_output=True, text=True)
    if r.returncode:
        raise RuntimeError(r.stdout + r.stderr)
    return os.path.join(pkg, "libapo_b200.so")


def phases(raw):
    """one launch's stamps [CTA][NSTAMP] -> microseconds after the earliest CTA entry (the latest of each phase)"""
    s = raw.reshape(MAX_CTAS, NSTAMP).astype(np.int64)
    live = s[:, 0] > 0
    t0 = s[live, 0].min()
    out = {}
    for i, name in enumerate(STAMPS):
        v = s[live, i]
        v = v[v > 0]
        out[name] = round(float(v.max() - t0) * 1e-3, 2) if len(v) else None
    out["ctas"] = int(live.sum())
    return out


def worker(lib, steps, warmup, diag):
    import importlib
    import torch
    eng_mod = importlib.import_module("senweaver-ide_b200.engine")
    eng_mod.LIB_PATH = lib
    pkg = importlib.import_module("senweaver-ide_b200")
    from form_d_tuple_copy import timed
    eng = pkg.Engine(0)
    out = {}
    try:
        stream = torch.cuda.current_stream()
        eng.set_stream(stream.cuda_stream)
        eng.dims_generate(SEED, 0, C, 0, T, 300)
        eng.corpus_generate(SEED, 0, T, 300)
        call = lambda: eng.score(C, K, corpus=True)
        tail = {"tail_finalize_ms": [], "tail_publish_ms": []}

        def call_tail():
            r = call()
            tail["tail_finalize_ms"].append(r.timing.tail_finalize_ms)
            tail["tail_publish_ms"].append(r.timing.tail_publish_ms)
            return r
        step, kern, r = timed(torch, eng, stream, call_tail, steps, warmup)
        out.update(step_ms=step, k1_ms=kern, host_gap_ms=[a - b for a, b in zip(step, kern)],
                   tail_finalize_ms=tail["tail_finalize_ms"][warmup:], tail_publish_ms=tail["tail_publish_ms"][warmup:])
        out["result"] = {"scores": r.scores.tolist(), "counts": r.counts.tolist(), "topk": r.topk.tolist()}
        if diag:
            L = ctypes.CDLL(lib)
            L.apo_diag_k1h_stamps.argtypes = [ctypes.c_void_p, ctypes.c_uint32]
            buf = np.zeros(MAX_CTAS * NSTAMP, np.uint64)
            ph = []
            for _ in range(steps):
                torch.cuda.synchronize()
                assert L.apo_diag_k1h_stamps(buf.ctypes.data, buf.size) == 0        # read and clear: the next call starts at zero
                call()
                torch.cuda.synchronize()
                assert L.apo_diag_k1h_stamps(buf.ctypes.data, buf.size) == 0
                ph.append(phases(buf))
            out["phases_us"] = ph
            os.environ["APO_K1H_DIAG"] = "1"
            for _ in range(warmup):
                call()
            out["stream_only_k1_ms"] = [call().timing.reward_ms for _ in range(steps)]
            os.environ["APO_K1H_DIAG"] = "0"
    finally:
        eng.close()
    print(json.dumps(out))


def run(lib, args, diag):
    cmd = [sys.executable, os.path.abspath(__file__), "--worker", lib, "--steps", str(args.steps), "--warmup", str(args.warmup)]
    if diag:
        cmd.append("--diag")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        raise RuntimeError(r.stderr[-4000:])
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--diag-lib")
    ap.add_argument("--lib", help="another build of the library for the plain part")
    ap.add_argument("--out")
    ap.add_argument("--worker")
    ap.add_argument("--diag", action="store_true")
    args = ap.parse_args()
    if args.worker:
        worker(args.worker, args.steps, args.warmup, args.diag)
        return
    from form_d_twin import card
    from form_d_tuple_copy import stats
    import importlib
    plain = importlib.import_module("senweaver-ide_b200.engine").LIB_PATH
    libs = {"this": plain} | ({"other": args.lib} if args.lib else {})
    with tempfile.TemporaryDirectory() as tmp:
        diag = args.diag_lib or build_diag(tmp)
        got = {name: [] for name in libs}
        dg = []
        for _ in range(args.rounds):
            for name, lib in libs.items():
                got[name].append(run(lib, args, False))
            dg.append(run(diag, args, True))
    out = {"card": card(), "workload": f"{C} x {T} Form D + {T}-record corpus (seed {SEED:#x}), apo_score with the corpus report, K={K}"}
    keys = ["step_ms", "k1_ms", "host_gap_ms", "tail_finalize_ms", "tail_publish_ms"]
    for name in libs:
        out[name] = {k: stats(sum((g[k] for g in got[name]), [])) for k in keys}
    if "other" in libs:
        a, b = got["this"][-1]["result"], got["other"][-1]["result"]
        out["same_result_as_other"] = a == b
    ph = sum((g["phases_us"] for g in dg), [])
    out["diag"] = {"phases_us_median": {k: round(float(np.median([p[k] for p in ph if p[k] is not None])), 2)
                                         for k in STAMPS if any(p[k] is not None for p in ph)},
                   "ctas": ph[0]["ctas"], "k1_ms": stats(sum((g["k1_ms"] for g in dg), [])),
                   "stream_only_k1_ms": stats(sum((g["stream_only_k1_ms"] for g in dg), []))}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
