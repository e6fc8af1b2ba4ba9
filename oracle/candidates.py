"""CPU oracle of the per-candidate breakdown (apo_candidate_report): ctypes front end of oracle/cand_oracle.c.

TEST INFRASTRUCTURE ONLY, like the rest of oracle/.  The C side returns exact integers; this module rounds each sum once
to binary64 (Python's int -> float conversion is correctly rounded, and the scaling by 2^-52 is exact) and applies the
report rules of APO:546-547, 556-568, 575, 591, 802, 819, the same rules the engine's corpus report applies.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from . import NDIM, RECORD_DTYPE, weights

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libcand_oracle.so")


class CandFx(C.Structure):
    _fields_ = [("total", C.c_uint64), ("good", C.c_uint64), ("bad", C.c_uint64), ("none", C.c_uint64), ("withReward", C.c_uint64),
                ("rew_lo", C.c_uint64), ("rew_hi", C.c_int64),
                ("dim_lo", C.c_uint64 * NDIM), ("dim_hi", C.c_int64 * NDIM), ("dim_count", C.c_uint64 * NDIM),
                ("badExamples", C.c_int64 * 3)]


def build(force: bool = False) -> str:
    src = [os.path.join(_HERE, f) for f in ("cand_oracle.c", "cand_oracle.h", "apo_oracle.c", "apo_oracle.h")]
    if force or not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in src):
        subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "candidates.mk", "libcand_oracle.so"])
    return _SO


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
        L.orc_cand_dims.argtypes = [vp, u32, u64, u64, u64, vp, vp]
        L.orc_cand_records.argtypes = [vp, u32, u64, u64, u64, vp, vp]
        L.orc_cand_generated.argtypes = [u64, vp, u32, u64, u64, u32, vp, vp, i32]
        L.orc_cand_generated_records.argtypes = [u64, vp, u32, u64, u64, u32, vp, vp, i32]
        for f in (L.orc_cand_dims, L.orc_cand_records, L.orc_cand_generated, L.orc_cand_generated_records):
            f.restype = None
        _lib = L
    return _lib


def _p(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def _i128(lo: int, hi: int) -> int:
    return (int(hi) << 64) + int(lo)


def fx_to_double(v: int) -> float:
    """Exact 2^-52 fixed point -> binary64 with one rounding (limbs_to_double)."""
    return float(v) * 2.0 ** -52


def dimstat(fx: int, count: int) -> dict:
    s = fx_to_double(fx)
    avg = s / count if count > 0 else 0.0                                        # APO:567
    return {"sum": s, "count": count, "avg": avg, "fx": fx,
            "low_flag": int(count >= 5 and avg < -0.3), "low_severity": 2 if avg < -0.5 else 1,       # APO:575, 591
            "sugg_flag": int(count >= 3 and avg < 0.0), "sugg_priority": 2 if avg < -0.5 else 1}      # APO:802, 819


def _report(r: CandFx) -> dict:
    good, bad, n = int(r.good), int(r.bad), int(r.withReward)
    rfx = _i128(r.rew_lo, r.rew_hi)
    rsum = fx_to_double(rfx)
    return {"total": int(r.total), "good": good, "bad": bad, "none": int(r.none),
            "goodRate": good / (good + bad) if good + bad > 0 else 0.0,                # APO:546-547
            "withReward": n, "rewardFx": rfx, "rewardSum": rsum, "avgReward": rsum / n if n > 0 else float("nan"),
            "dim": [dimstat(_i128(r.dim_lo[i], r.dim_hi[i]), int(r.dim_count[i])) for i in range(NDIM)],
            "badExamples": [int(x) for x in r.badExamples]}


def cand_dims(dims: np.ndarray, T: int | None = None, idx_base: int = 0, w=None) -> list[dict]:
    """dims float32 [C][pitch][9] -> one breakdown dict per candidate over records [0, T)."""
    dims = np.ascontiguousarray(dims, np.float32)
    Cn, pitch, nd = dims.shape
    assert nd == NDIM
    T = pitch if T is None else T
    w = weights() if w is None else np.ascontiguousarray(w, np.float64)
    out = (CandFx * Cn)()
    lib().orc_cand_dims(_p(dims), Cn, T, pitch, idx_base, _p(w), out)
    return [_report(r) for r in out]


def cand_records(recs: np.ndarray, T: int | None = None, idx_base: int = 0, w=None) -> list[dict]:
    """Form R [C][pitch] -> one breakdown dict per candidate (the corpus report of each row, on the shared fields)."""
    recs = np.ascontiguousarray(recs, RECORD_DTYPE)
    Cn, pitch = recs.shape
    T = pitch if T is None else T
    w = weights() if w is None else np.ascontiguousarray(w, np.float64)
    out = (CandFx * Cn)()
    lib().orc_cand_records(_p(recs), Cn, T, pitch, idx_base, _p(w), out)
    return [_report(r) for r in out]


def cand_generated(seed: int, cands, t0: int, T: int, agent_permille: int = 300, w=None, nthreads: int = 8,
                   records: bool = False) -> list[dict]:
    """Breakdown of the listed candidates over generated evaluations [t0, t0+T), generated on the fly: Form D rows, or with
    records=True the rollout records themselves (what apo_rollouts_generate / apo_rollouts16_generate load)."""
    cands = np.ascontiguousarray(cands, np.uint32)
    w = weights() if w is None else np.ascontiguousarray(w, np.float64)
    out = (CandFx * len(cands))()
    f = lib().orc_cand_generated_records if records else lib().orc_cand_generated
    f(seed, _p(cands), len(cands), t0, T, agent_permille, _p(w), out, nthreads)
    return [_report(r) for r in out]
