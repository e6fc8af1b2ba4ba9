"""Where K1t2's time goes on the flagship tensor (256 x 5 M Form D, seed 0x5EED0003: the configs[2] step's scoring kernel).

Times, with CUDA events (apo_last_timing's kernel time) over --steps launches each, alternating in rounds:
  slots      K1t2 as built: the slot plane, the slot-order head in shared memory, the tail through L2, both lists
  stream     the stream alone: the raw slots are added (no gather)
  head       the gather clamped to the shared-memory head (no ld.global)
  other      K1t2 of another build of the library (--other-lib, e.g. the previous commit's: the dictionary-index plane)
The stream and head variants exist only in a build with -DAPO_K1T2_DIAG (their sums are not the table's); the script
compiles one into a temporary directory unless --diag-lib names one.  It also prints the wavefront model
(tests/slot_model.py) of the flagship's first --model-rows rows x 1 M evaluations for the plain index plane and for the
slot plane: distinct 4-byte words per bank of each warp instruction, over the warp and per half-warp, and the lanes that
take the L2 path.

    python examples/k1t2_gather.py [--steps 60] [--rounds 3] [--diag-lib SO] [--other-lib SO] [--model-rows 4] [--out FILE]

Prints one JSON object with the card's name and power limit read in the same run."""
import argparse
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
SEED, C, T, K = 0x5EED0003, 256, 5_000_000, 64
MODES = {"slots": "0", "stream": "1", "head": "2"}


def build_diag(tmp):
    """the library with the diagnostic variants, compiled from this tree's sources into tmp"""
    src = os.path.join(ROOT, "senweaver-ide_b200", "csrc")
    pkg = os.path.join(tmp, "pkg")
    shutil.copytree(src, os.path.join(pkg, "csrc"), ignore=shutil.ignore_patterns("*.o"))
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(tmp, "include"))
    r = subprocess.run(["make", "-s", "-C", os.path.join(pkg, "csrc"), "NVCC=nvcc -DAPO_K1T2_DIAG"], capture_output=True, text=True)
    if r.returncode:
        raise RuntimeError(r.stdout + r.stderr)
    return os.path.join(pkg, "libapo_b200.so")


def worker(lib, modes, steps, warmup, model_rows):
    """one process on one library: the flagship tensor, then `steps` K1t2 launches per mode"""
    import importlib
    import torch
    eng_mod = importlib.import_module("senweaver-ide_b200.engine")
    eng_mod.LIB_PATH = lib
    pkg = importlib.import_module("senweaver-ide_b200")
    eng = pkg.Engine(0)
    out = {}
    try:
        stream = torch.cuda.current_stream()
        eng.set_stream(stream.cuda_stream)
        eng.dims_generate(SEED, 0, C, 0, T, 300)
        for name in modes:
            os.environ["APO_K1T2_DIAG"] = MODES.get(name, "0")
            for _ in range(warmup):
                eng.score(C, K)
            ms = []
            for _ in range(steps):
                ms.append(eng.score(C, K).timing.reward_ms)
            out[name] = ms
        os.environ["APO_K1T2_DIAG"] = "0"
        if model_rows:
            out["model"] = model(eng, model_rows)
    finally:
        eng.close()
    print(json.dumps(out))


def model(eng, rows):
    import slot_model as sm
    n = eng.dims_tuples()                                 # resident Form T of the tensor: the copy's dictionary
    idx = np.empty((rows, 1 << 20), np.int64)
    for c in range(rows):
        lo, hi = eng.tuples_download(c, 0, 1 << 20)
        idx[c] = lo.astype(np.int64) | (hi.astype(np.int64) << 16)
    h = min(sm.SLOT_H, n)                                 # build_twin_t2 keeps it unless the second list grows past 1/64
    end = sm.slot_end(n, h)
    out = {"distinct": int(n), "h": h, "end": end,
           "share_below_24576": float((idx < 24576).mean()), "share_below_2^16": float((idx < 65536).mean()),
           "share_listed": float((idx >= end).mean()),
           "index_plane": sm.wavefronts(idx & 0xFFFF, hot=24576),
           "slot_plane": sm.wavefronts(sm.slot_plane(idx, h, end))}
    return out


def run(lib, modes, args, model_rows=0):
    cmd = [sys.executable, os.path.abspath(__file__), "--worker", lib, "--modes", ",".join(modes), "--steps", str(args.steps),
           "--warmup", str(args.warmup), "--model-rows", str(model_rows)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        raise RuntimeError(r.stderr[-4000:])
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--diag-lib")
    ap.add_argument("--other-lib")
    ap.add_argument("--model-rows", type=int, default=4)
    ap.add_argument("--out")
    ap.add_argument("--worker")
    ap.add_argument("--modes")
    args = ap.parse_args()
    if args.worker:
        worker(args.worker, args.modes.split(","), args.steps, args.warmup, args.model_rows)
        return
    from form_d_twin import card
    from form_d_tuple_copy import stats
    with tempfile.TemporaryDirectory() as tmp:
        diag = args.diag_lib or build_diag(tmp)
        times = {m: [] for m in list(MODES) + (["other"] if args.other_lib else [])}
        model_out = None
        for rnd in range(args.rounds):
            got = run(diag, list(MODES), args, args.model_rows if rnd == 0 else 0)
            model_out = got.pop("model", model_out)
            for m, v in got.items():
                times[m] += v
            if args.other_lib:
                times["other"] += run(args.other_lib, ["other"], args)["other"]
    out = {"card": card(), "workload": f"{C} x {T} Form D (seed {SEED:#x}), apo_score K={K} without the corpus: one K1t2 launch",
           "timing": "kernel time from apo_last_timing (CUDA events around the launch)",
           "kernel_ms": {m: stats(v) for m, v in times.items()}, "model": model_out,
           "bytes_per_eval_stream": 2.0, "hbm_floor_ms_at_3350GBps": round(2.0 * C * T / 3.35e12 * 1e3, 4)}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
