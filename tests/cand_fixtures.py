"""Hand-built Form D tensors that reach the edges of the per-candidate breakdown (csrc/apo_cand.cu k_cand_breakdown /
k_cand_report), and an exact pure-Python model of the breakdown they are checked against.

Every fixture holds at most 15 values per coded dimension and at most 4095 tool_success_rate values, so the same tensor goes
through every loader (Form D, the Form W / Q copies, Form P, the Form T dictionary).  Large values sit in dimensions of
weight 0 (W_BIG: d0, d3, d4, d8), so that finalReward stays inside Form T's (-2, 2) domain while the dimension sums grow.

- large_sums: dimension sums past 2^64 and 2^83 in both signs (values +-1024 and +-(2048 - 2^-13), the largest magnitude
  with an exact term, over 2^20 + 33 counted evaluations per candidate), and rows whose halves cancel, across warps, to exactly
  0, to +-1 unit and to +-2^64.
- ties: dimension sums (2^53 + 1) * 2^k with and without a sticky unit, below 2^64 (the (double)lo branch of
  limbs_to_double) and at or above it (the top-64-bits-plus-sticky branch), in both signs; and fp32 values whose v * 2^52
  is k + 1/2 (2^-53, 3 * 2^-53, 5 * 2^-53, both signs) and the subnormal 1e-45, for rint's ties to even in to_fx.
- report_rules: dimension averages exactly RN(-0.3), -0.5 and 0.0 and one step to each side, at counts 2 ... 5, across the
  thresholds of low_flag / low_severity / sugg_flag / sugg_priority.
- tallies: d0 = +-1 (good / bad), +-nextafter(1) (none), absent (none), null evaluations with d0 = -1 (bad, in no sum),
  zero-weight masks beside masks whose total weight has an all-ones significand; goodRate at good = bad, good = 0, bad = 0.
- shapes: rows of T = 1024 + r, r in {1, 31, 32, 33, 127, 128, 129, 1023}, and 600 candidates of T = 33, so one warp walks
  many candidates.
- domain_*: the values 2048, -2048, 3000, 1e30 and 2048 - 2^-13 in a counted evaluation, in a null evaluation and in d0, and
  d3 = 3000 with d4 = -4800 under the default weights (finalReward ~ 0): a call with APO_SCORE_CANDIDATES refuses every
  counted |v| >= 2048 and accepts the rest exactly.

Plain helpers (no pytest fixtures, no GPU)."""
from __future__ import annotations

from fractions import Fraction

import numpy as np

import oracle

FX = 1 << 52
NAN = np.float32("nan")
BIG = float(2048 - 2.0 ** -13)                   # largest fp32 below 2048: its term 2^63 - 2^39 is the largest exact one
W_BIG = np.array([0.0, 0.25, 0.25, 0.0, 0.0, 0.25, 0.125, 0.125 - 2.0 ** -53, 0.0])   # {1,2,5,6,7}: tw = 1 - 2^-53
LARGE_T = (1 << 20) + 33
SHAPE_TAILS = (1, 31, 32, 33, 127, 128, 129, 1023)


def rows(n: int, **dims) -> np.ndarray:
    """n evaluations with dimension i = dims[f'd{i}'] (scalar or array), every other dimension absent"""
    r = np.full((n, 9), NAN, np.float32)
    for k, v in dims.items():
        r[:, int(k[1:])] = v
    return r


def base(n: int) -> np.ndarray:
    """n counted evaluations (d1 = 0.5 carries weight) with nothing else present"""
    return rows(n, d1=0.5)


# ------------------------------------------------------------------------------------------------ fixtures
def large_sums() -> np.ndarray:
    """[4][2^20 + 33][9]: c0 / c1 all one sign (d3 ~ +-2^83, d4 ~ -+2^82, d8 ~ +-2^64 + ...); c2 / c3 halves that cancel"""
    T, h = LARGE_T, LARGE_T // 2
    d = np.repeat(base(T)[None], 4, axis=0)
    d[:, :, 0] = np.where(np.arange(T) % 3 == 0, 1.0, -1.0)                     # tallies on the way
    for c, s in ((0, 1.0), (1, -1.0)):
        d[c, :, 3] = s * BIG
        d[c, :, 4] = -s * 1024.0
        d[c, :, 8] = s * 2.0 ** -40                                             # 2^12 units per evaluation: ~2^32, one limb up
    for c, s in ((2, 1.0), (3, -1.0)):
        d[c, :h, 3], d[c, h:2 * h, 3] = BIG, -BIG                               # exactly 0 (+0.0 expected: sugg_flag 0)
        d[c, 2 * h:, 3] = np.nan
        d[c, :h, 4], d[c, h:2 * h, 4] = 1024.0, -1024.0
        d[c, 2 * h:, 4] = np.nan
        d[c, T - 1, 4] = s * 2.0 ** -52                                         # +-1 unit
        d[c, :h, 8], d[c, h:2 * h - 4, 8] = s * 1024.0, -s * 1024.0             # four more of one sign: +-2^64
        d[c, 2 * h - 4:, 8] = np.nan
    return d


TIE_SUMS = {                                                                    # fx units: value of the rows below
    "lo_tie": (1 << 60) + (1 << 7),                                             # (2^53 + 1) * 2^7: even -> 2^60
    "lo_sticky": (1 << 60) + (1 << 7) + 1,
    "hi_tie": (1 << 64) + (1 << 11),                                            # (2^53 + 1) * 2^11: even -> 2^64
    "hi_sticky": (1 << 64) + (1 << 11) + 1,
}
TIE_VALUES = (2.0 ** -53, 3 * 2.0 ** -53, 5 * 2.0 ** -53, -(2.0 ** -53), -3 * 2.0 ** -53, -5 * 2.0 ** -53, float(np.float32(1e-45)))


def ties() -> np.ndarray:
    """[8][129][9]: candidate 2k / 2k+1 hold TIE_SUMS[k] / its negation in d3 (from 256, 1024, 2^-45, 2^-41, 2^-52), and
    every candidate the to_fx ties TIE_VALUES in d4, one per evaluation"""
    T = 129
    d = np.repeat(base(T)[None], 8, axis=0)
    parts = {"lo_tie": [256.0, 2.0 ** -45], "lo_sticky": [256.0, 2.0 ** -45, 2.0 ** -52],
             "hi_tie": [1024.0] * 4 + [2.0 ** -41], "hi_sticky": [1024.0] * 4 + [2.0 ** -41, 2.0 ** -52]}
    for k, name in enumerate(TIE_SUMS):
        for c, s in ((2 * k, 1.0), (2 * k + 1, -1.0)):
            v = np.array(parts[name]) * s
            d[c, 40:40 + len(v), 3] = v                                         # in the second 32-group, across lanes
            d[c, :, 4] = np.resize(np.array(TIE_VALUES, np.float32), T)
    return d


REPORT_TARGETS = (-0.3, -0.5, 0.0)
REPORT_PALETTE = (-0.5, -0.25, -0.375, -0.125, 0.0, 2.0 ** -52, -(2.0 ** -52), 2.0 ** -51, -(2.0 ** -51), 0.25, -0.75)


def _avg(vals) -> float:
    """the breakdown's average of fp32 values vals: RN(RN(sum) / count)"""
    S = sum(round(Fraction(float(np.float32(v))) * FX) for v in vals)
    return float(Fraction(S, FX)) / len(vals)


def report_rows() -> list[tuple]:
    """(values, average) for every count 2 ... 5 and every target t in REPORT_TARGETS: the first multiset of REPORT_PALETTE
    (in a fixed enumeration order) whose average is t, nextafter(t, -inf) and nextafter(t, +inf) (for 0.0: the nearest
    averages a sum of +-1 unit gives), where one exists"""
    from itertools import combinations_with_replacement
    out = []
    for n in (2, 3, 4, 5):
        found = {}
        for vals in combinations_with_replacement(REPORT_PALETTE, n):
            a = _avg(vals)
            for t in REPORT_TARGETS:
                lo = -(2.0 ** -52) / n if t == 0.0 else float(np.nextafter(t, -np.inf))
                hi = (2.0 ** -52) / n if t == 0.0 else float(np.nextafter(t, np.inf))
                for want in (lo, t, hi):
                    if a == want and (t, want) not in found:
                        found[(t, want)] = vals
        out += [(vals, want) for (t, want), vals in sorted(found.items())]
    return out


def report_rules() -> np.ndarray:
    """one candidate per report_rows() entry: its values in d5 (weight 0.25) over evaluations 0 .. n-1 of a row of T = 32"""
    R = report_rows()
    d = np.repeat(base(32)[None], len(R), axis=0)
    for c, (vals, _) in enumerate(R):
        d[c, :len(vals), 5] = vals
    return d


D0_NEXT = float(np.nextafter(np.float32(1), np.float32(2)))


def tallies() -> np.ndarray:
    """[5][64][9] (W_BIG): c0 good = bad; c1 good = 0, with null evaluations among the counted ones; c2 bad = 0; c3 nothing
    but none; c4 only null evaluations (d0 = -1 with d3 alone, weight 0), so bad > 0 and withReward = 0.  Masks: {1,2,5,6,7} (tw = 1 - 2^-53) beside {3} (tw = 0)"""
    T = 64
    full = rows(T, d1=0.25, d2=0.5, d5=-0.5, d6=0.75, d7=-0.25)
    d = np.repeat(full[None], 5, axis=0)
    d[0, :, 0] = np.resize(np.array([1.0, -1.0, D0_NEXT, -D0_NEXT, NAN], np.float32), T)
    d[1, :, 0] = np.resize(np.array([-1.0, NAN, -D0_NEXT], np.float32), T)
    d[2, :, 0] = np.resize(np.array([1.0, D0_NEXT, 0.5], np.float32), T)
    d[3, :, 0] = np.resize(np.array([NAN, D0_NEXT, -D0_NEXT, 0.0], np.float32), T)
    d[4] = rows(T, d0=-1.0, d3=0.5)                                             # zero total weight: null, tallied bad
    d[1, 5::7] = rows(len(range(5, T, 7)), d0=-1.0, d3=0.75)                    # null evaluations among counted ones
    return d


def shapes(tail: int) -> np.ndarray:
    """[3][1024 + tail][9]: categorical values with holes (palettes of <= 12 values per dimension, d2 of 100)"""
    return categorical(0x5EEDCA00 + tail, 3, 1024 + tail)


def many_short() -> np.ndarray:
    """[600][33][9]: one warp's tile range crosses many candidates"""
    return categorical(0x5EEDCA01, 600, 33)


def categorical(seed: int, C: int, T: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    pal = np.array([-1.0, -0.75, -0.5, -0.25, 0.0, 0.25, 0.5, 0.75, 1.0, 0.125, -0.125, 2.0 ** -53], np.float32)
    d = pal[rng.integers(0, len(pal), (C, T, 9))]
    d[:, :, 0] = np.array([1.0, -1.0, D0_NEXT, 0.5], np.float32)[rng.integers(0, 4, (C, T))]
    d[:, :, 2] = rng.uniform(0, 1, 100).astype(np.float32)[rng.integers(0, 100, (C, T))]
    d[rng.random((C, T, 9)) < 0.15] = np.nan
    return d


DOMAIN_VALUES = (2048.0, -2048.0, 3000.0, 1e30, BIG)


def domain(value: float, where: str) -> tuple[np.ndarray, np.ndarray]:
    """(dims [2][40][9], weights): `value` at candidate 1, evaluation 37, in d4 of a counted evaluation ('counted'), in d4 of
    a null one ('null': only weight-0 dimensions present), in d0 of a counted one ('d0'); 'pair': d3 = 3000 and d4 = -4800
    beside d1 under the default weights"""
    d = np.repeat(base(40)[None], 2, axis=0)
    d[:, :, 4] = 0.5
    if where == "pair":
        d[1, 37, 3], d[1, 37, 4] = 3000.0, -4800.0
        return d, oracle.weights()
    if where == "counted":
        d[1, 37, 4] = value
    elif where == "null":
        d[1, 37] = rows(1, d3=0.5, d4=value)[0]
    elif where == "d0":
        d[1, 37, 0] = value
    else:
        raise ValueError(where)
    return d, W_BIG


def domain_refused(value: float, where: str) -> bool:
    return where == "pair" or (where != "null" and abs(value) >= 2048.0)


def domain_cases():
    return [(v, w) for v in DOMAIN_VALUES for w in ("counted", "null", "d0")] + [(3000.0, "pair")]


# ------------------------------------------------------------------------------------------------ exact model
def _final_rewards(d: np.ndarray, w: np.ndarray):
    """TCS:784 in binary64, in dimension order, as orc_final_reward: (valid, finalReward) per evaluation"""
    ws = np.zeros(d.shape[:-1])
    tw = np.zeros(d.shape[:-1])
    for i in range(9):
        p = ~np.isnan(d[..., i])
        ws = np.where(p, ws + d[..., i].astype(np.float64) * w[i], ws)
        tw = np.where(p, tw + w[i], tw)
    valid = tw > 0
    with np.errstate(invalid="ignore", divide="ignore"):
        return valid, np.where(valid, ws / np.where(valid, tw, 1.0), 0.0)


def _fx_sum(values: np.ndarray) -> int:
    """exact sum of rint(v * 2^52) (ties to even) over fp32 values, by distinct value"""
    u, n = np.unique(values.astype(np.float64), return_counts=True)
    return sum(int(k) * round(Fraction(float(v)) * FX) for v, k in zip(u, n))


def exact_breakdown(d: np.ndarray, w=None, idx_base: int = 0) -> tuple[list[dict], bool]:
    """(breakdown per candidate, refused): the report fields in plain Python (Fraction -> float, one rounding per sum),
    with the terms of counted |v| >= 2048 left out and refused = True when there is one"""
    w = oracle.weights() if w is None else np.asarray(w, np.float64)
    valid, fr = _final_rewards(d, w)
    refused = False
    out = []
    for c in range(d.shape[0]):
        v, x = valid[c], d[c]
        d0 = x[:, 0]
        good, bad = int((d0 == 1.0).sum()), int((d0 == -1.0).sum())
        r = {"total": x.shape[0], "good": good, "bad": bad, "none": x.shape[0] - good - bad,
             "goodRate": good / (good + bad) if good + bad else 0.0, "withReward": int(v.sum())}
        rfx = sum(int(k) * int(np.rint(f * FX)) for f, k in zip(*np.unique(fr[c][v], return_counts=True)))
        r["rewardFx"] = rfx
        r["rewardSum"] = float(Fraction(rfx, FX))
        r["avgReward"] = r["rewardSum"] / r["withReward"] if r["withReward"] else float("nan")
        dims = []
        for i in range(9):
            col = x[v, i]
            col = col[~np.isnan(col)]
            big = np.abs(col.astype(np.float64)) >= 2048.0
            refused |= bool(big.any())
            col = col[~big]
            fx = _fx_sum(col) if len(col) else 0
            s = float(Fraction(fx, FX))
            n = len(col)
            avg = s / n if n else 0.0
            dims.append({"sum": s, "count": n, "avg": avg, "fx": fx,
                         "low_flag": int(n >= 5 and avg < -0.3), "low_severity": 2 if avg < -0.5 else 1,
                         "sugg_flag": int(n >= 3 and avg < 0.0), "sugg_priority": 2 if avg < -0.5 else 1})
        r["dim"] = dims
        ex = [idx_base + int(t) for t in np.flatnonzero(d0 == -1.0)[:3]]
        r["badExamples"] = ex + [-1] * (3 - len(ex))
        out.append(r)
    return out, refused
