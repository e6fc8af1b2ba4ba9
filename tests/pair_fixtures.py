"""Form D tensors and reference lists that reach the edges of the paired comparison (csrc/apo_cand.cu k_cand_pairs /
k_cand_pair_report), and the exact integer model the engine is checked against.

For candidate c with reference r = refs[c], x_t = rint(fr_t * 2^52) of the non-null evaluations (fr_t as
extremes_fixtures.final_rewards / record_final_rewards restate the scoring arithmetic), over the positions where both rows
have a finalReward, d_t = x_c,t - x_r,t:
    n, wins / losses / ties (d > 0 / < 0 / == 0), candOnly / refOnly (only one row non-null),
    D1 = sum d_t, D2 = sum d_t^2, M = n * D2 - D1^2,
    meanDiff = RN(D1) * 2^-52 / (double)n (NaN when n == 0), and variance / stdDev / stdErr by the spread's rules
    (spread_fixtures.fields with D1, D2 for S1, S2).
Python's float(int) is correctly rounded and math.ldexp, / and math.sqrt are IEEE operations, so the model reproduces
every bit.

Fixtures (each weighs d1 alone with weight 1.0 unless it says otherwise, so that fr = v exactly and x = v * 2^52):
- extreme: c at fr = 512 - 2^-15 against r at fr = -512 over 2^22 + 3 evaluations: |d| = 2^62 - 2^37, D1 passes 2^64 and
  2^83, D2 passes 2^128.  Refs [1, 0] give the pair and its mirror, refs [0, 1] two self-pairs.  Only Form D through K1 and
  the Form W / Q copy admit it (the Form T copy's domain is (-2, 2)); extreme(T) is the same at a smaller T.
- one_unit: rows at fr = 1.5, with one evaluation one unit (2^-52) lower at a chosen position (d2 = 0 present under
  w_one_unit): the smallest win and loss.
- nulls: generator rows whose last evaluation (T mod 1024 in TAILS) and chosen others are null on either side.
- rn_edges: spread_fixtures.rn_edges rows against a row at fr = 0: M = p q m^2 meets the four RN(M) edges.
- counts: n = 0, 1, 2.
- shapes: many candidates naming one reference, references of higher and lower index, a chain a -> b -> c, a self-pair
  and candidates without a reference.

Plain helpers (no pytest fixtures, no GPU)."""
from __future__ import annotations

import math

import numpy as np

import oracle
import spread_fixtures as sf
from extremes_fixtures import NAN, final_rewards, record_final_rewards, rows

NONE = 0xFFFFFFFF
TAILS = sf.TAILS
FIELDS = ("ref", "n", "wins", "losses", "ties", "candOnly", "refOnly", "sumLo", "sumHi", "sumSq0", "sumSq1", "sumSq2",
          "meanDiff", "variance", "stdDev", "stdErr")


# ------------------------------------------------------------------------------------------------ the model
def xterms(fr: np.ndarray, ok: np.ndarray) -> np.ndarray:
    """rint(fr * 2^52) of every evaluation as int64 (0 where null)"""
    return np.rint(np.where(ok, np.asarray(fr, np.float64), 0.0) * sf.FX).astype(np.int64)


def pair_fields(ref: int, n: int, wins: int, losses: int, ties: int, c_only: int, r_only: int, d1: int, d2: int) -> dict:
    """one apo_candidate_pair from its integers, with the header's sequence of operations"""
    s = sf.fields(n, d1, d2)
    out = {"ref": ref, "n": n, "wins": wins, "losses": losses, "ties": ties, "candOnly": c_only, "refOnly": r_only,
           "sumLo": d1 & (2 ** 64 - 1), "sumHi": d1 >> 64, "sumSq0": s["sumSq0"], "sumSq1": s["sumSq1"], "sumSq2": s["sumSq2"],
           "meanDiff": s["mean"], "variance": s["variance"], "stdDev": s["stdDev"], "stdErr": s["stdErr"], "D1": d1, "D2": d2,
           "M": s["M"]}
    return out


def none_fields() -> dict:
    return pair_fields(NONE, 0, 0, 0, 0, 0, 0, 0, 0)


def pair_model(fr, ok, refs) -> list[dict]:
    """pairs of rows fr / ok [C][T] under refs [C]"""
    fr, ok = np.atleast_2d(fr), np.atleast_2d(ok).astype(bool)
    x = xterms(fr, ok)
    out = []
    for c, r in enumerate(int(v) for v in refs):
        if r == NONE:
            out.append(none_fields())
            continue
        both = ok[c] & ok[r]
        d = x[c][both] - x[r][both]                      # |d| <= 2^62: exact in int64
        do = d.astype(object)
        out.append(pair_fields(r, int(d.size), int((d > 0).sum()), int((d < 0).sum()), int((d == 0).sum()),
                               int((ok[c] & ~ok[r]).sum()), int((ok[r] & ~ok[c]).sum()),
                               int(do.sum()) if d.size else 0, int((do * do).sum()) if d.size else 0))
    return out


def model(dims: np.ndarray, refs, w=None, recip: bool = False) -> list[dict]:
    """pairs of Form D dims [C][T][9] scored whole"""
    return pair_model(*final_rewards(dims, w, recip), refs)


def rec_model(recs: np.ndarray, refs, w=None, recip: bool = False) -> list[dict]:
    return pair_model(*record_final_rewards(recs, w, recip), refs)


def constant_pair(n: int, vc: float, vr: float, ref: int) -> dict:
    """n positions with c at fr = vc and r at fr = vr (v * 2^52 integers)"""
    xc, xr = int(vc * sf.FX), int(vr * sf.FX)
    d = xc - xr
    return pair_fields(ref, n, n if d > 0 else 0, n if d < 0 else 0, n if d == 0 else 0, 0, 0, n * d, n * d * d)


def fraction_sums(fr, ok, c: int, r: int):
    """(D1, D2) of the pair (c, r) by exact rational arithmetic on the finalRewards themselves"""
    from fractions import Fraction
    fr, ok = np.atleast_2d(fr), np.atleast_2d(ok)
    s1 = s2 = Fraction(0)
    for fc, fr_, a, b in zip(fr[c].tolist(), fr[r].tolist(), ok[c].tolist(), ok[r].tolist()):
        if a and b:
            d = Fraction(round(Fraction(fc) * 2 ** 52)) - Fraction(round(Fraction(fr_) * 2 ** 52))
            s1 += d
            s2 += d * d
    return int(s1), int(s2)


# ------------------------------------------------------------------------------------------------ fixtures
def extreme(T: int = (1 << 22) + 3) -> np.ndarray:
    """[2][T][9]: row 0 at 512 - 2^-15, row 1 at -512"""
    return np.stack([rows(T, d1=np.float32(sf.F32_BELOW_512)), rows(T, d1=np.float32(-512.0))])


def one_unit(T: int = 4096 + 33, at=(1500, 3001)) -> np.ndarray:
    """[3][T][9] under sf.w_one_unit: d1 = 1.5 everywhere; row 1 one unit lower at at[0], row 2 at at[1]"""
    d = np.stack([rows(T, d1=np.float32(1.5)) for _ in range(3)])
    d[1, at[0], 2] = 0.0
    d[2, at[1], 2] = 0.0
    return d


ONE_UNIT_REFS = np.array([1, 0, 1], np.uint32)           # a win, a loss, and a win and a loss in one pair


def nulls(seed: int = 5):
    """one [2][T][9] generator tensor per T = 1024 + r, r in TAILS: row 0's last evaluation null, row 1's first and a middle
    one null, every 7th null in both"""
    out = []
    for r in TAILS:
        T = 1024 + r
        d = oracle.gen_dims(0x5EED7200 + seed, 0, 2, 0, T, 300, 4)
        d[0, T - 1] = NAN
        d[1, 0] = NAN
        d[1, T // 2] = NAN
        d[:, ::7] = NAN
        out.append(d)
    return out


NULL_REFS = np.array([1, 0], np.uint32)


def rn_edges() -> np.ndarray:
    """[5][RN_T][9]: spread_fixtures.rn_edges and a row at fr = 0 over every position"""
    return np.concatenate([sf.rn_edges(), rows(sf.RN_T, d1=np.float32(0))[None]])


RN_REFS = np.array([4, 4, 4, 4, NONE], np.uint32)


def counts(T: int = 2 * 1024 + 33) -> np.ndarray:
    """[4][T][9]: row 0 all null; row 1 valid at 700 only, row 2 at 5 and T - 1, row 3 everywhere (alternating +-1)"""
    d = np.full((4, T, 9), NAN, np.float32)
    d[1, 700, 1] = 0.25
    d[2, 5, 1], d[2, T - 1, 1] = -0.5, 0.375
    d[3, :, 1] = np.where(np.arange(T) % 2 == 0, 1.0, -1.0)
    return d


COUNT_REFS = np.array([3, 3, 3, 0], np.uint32)           # n = 0, 1, 2, and 0 again (refOnly = 0, candOnly = T)


def shapes(T: int = 3 * 1024 + 77, seed: int = 7) -> np.ndarray:
    d = oracle.gen_dims(0x5EED7300 + seed, 0, 8, 0, T, 300, 4)
    d[:, ::11] = NAN
    return d


# 1, 2, 3 name 0 (higher naming lower); 4 -> 5 -> 6 a chain (lower naming higher); 6 none; 7 itself; 0 none
SHAPE_REFS = np.array([NONE, 0, 0, 0, 5, 6, NONE, 7], np.uint32)


def all_fixtures():
    """(name, dims, refs, w) of every fixture above but the 2^22-row extreme one"""
    out = [("extreme_small", extreme(8192 + 5), np.array([1, 0], np.uint32), sf.w_one()),
           ("one_unit", one_unit(), ONE_UNIT_REFS, sf.w_one_unit()), ("rn_edges", rn_edges(), RN_REFS, sf.w_one()),
           ("counts", counts(), COUNT_REFS, sf.w_one()), ("shapes", shapes(), SHAPE_REFS, None)]
    out += [(f"nulls_{d.shape[1]}", d, NULL_REFS, None) for d in nulls()]
    return out


def invariants(p, counts_, partial_sums=None, nulls_free=None):
    """the relations every pair of a call satisfies against the call's counts (and, where neither row has a null,
    apo_debug_partials' S1): returns nothing, asserts"""
    for c, x in enumerate(p):
        r = int(x.ref)
        if r == NONE:
            assert (x.n, x.wins, x.losses, x.ties, x.candOnly, x.refOnly, x.sum, x.sum_sq) == (0,) * 8, c
            assert math.isnan(x.meanDiff) and math.isnan(x.variance), c
            continue
        assert x.n + x.candOnly == counts_[c] and x.n + x.refOnly == counts_[r], c
        assert x.wins + x.losses + x.ties == x.n, c
        if r == c:
            assert x.ties == x.n and x.sum == 0 and x.sum_sq == 0, c
        if partial_sums is not None and nulls_free is not None and nulls_free[c] and nulls_free[r]:
            assert x.sum == partial_sums[c] - partial_sums[r], c
        m = p[r] if int(p[r].ref) == c else None      # the mirror, when r names c
        if m is not None:
            assert (m.n, m.sum_sq, m.wins, m.losses, m.candOnly, m.refOnly, m.sum) == \
                (x.n, x.sum_sq, x.losses, x.wins, x.refOnly, x.candOnly, -x.sum), c
            assert np.float64(m.variance).tobytes() == np.float64(x.variance).tobytes(), c
