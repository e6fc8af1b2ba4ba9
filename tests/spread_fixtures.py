"""Form D tensors that reach the edges of the per-candidate reward spread (csrc/apo_cand.cu k_cand_spread /
k_cand_spread_report), and the exact model the engine is checked against.

For candidate c, over the evaluations the scoring call summed into scores[c] (x_t = rint(fr_t * 2^52), fr_t as
extremes_fixtures.final_rewards / record_final_rewards restate the scoring arithmetic):
    n = counts[c],  S1 = sum x_t,  S2 = sum x_t^2,  M = n * S2 - S1^2
and the binary64 fields are built with the operations the header states (RN = round to nearest even; Python's float(int)
is correctly rounded, and math.ldexp, / and math.sqrt are IEEE operations, so the model reproduces every bit):
    mean = RN(S1) * 2^-52 / (double)n (scores[c]; NaN when n == 0), rewardSumSq = RN(S2) * 2^-104,
    variance = RN(RN(RN(M) * 2^-104 / n) / (n - 1)) (NaN when n < 2), stdDev = sqrt(variance), stdErr = sqrt(RN(variance / n)).

Fixtures (each weighs d1 alone with weight 1.0 unless it says otherwise, so that fr = v exactly and x = v * 2^52):
- const512: rows at fr = -512 (x = -2^61) and at 512 - 2^-15, the largest fp32 below 512; 8192 + 5 evaluations, so a lane's
  sum passes 2^128 inside one run (256 terms of 2^122) and M = 0 exactly: every spread field is +0.0.  Only Form D through K1
  and the Form W / Q copy admit them; the Form T copy's domain is (-2, 2).
- const2: fr = -(2 - 2^-23), the edge of the Form T domain: x^2 ~ 2^106 passes 2^64 in every term.  2^128 is passed only
  over a whole row of >= 2^22 evaluations (const2_wide, a GPU-sized row).
- one_unit: equal rows at fr = 1.5 but one evaluation 2^-52 lower (d2 = 0 present with weight 2^-52, so its total weight is
  1 + 2^-52): its term is one unit below the others and M = n - 1 exactly, a tiny result of sums near 2^105 * n.
- rn_edges: rows of p terms m and q terms 0, so M = p q m^2; m is chosen so that RN(M) meets a tie that rounds to even
  downwards, a tie that rounds up, a value a sticky bit above half an ulp, and one below.
- counts: n = 0, 1, 2 (NaN / NaN / defined); null evaluations interleaved; alternating +-1 (variance n / (n - 1) rounded).
- tails: generator rows that end at T mod 1024 in TAILS, under the default weights.

Plain helpers (no pytest fixtures, no GPU)."""
from __future__ import annotations

import math

import numpy as np

import oracle
from extremes_fixtures import NAN, final_rewards, record_final_rewards, rows

FX = float(2 ** 52)
TAILS = (1, 31, 32, 33, 127, 128, 129, 1023)
F32_BELOW_512 = float(np.nextafter(np.float32(512), np.float32(0)))       # 512 - 2^-15
F32_BELOW_2 = float(np.nextafter(np.float32(2), np.float32(0)))           # 2 - 2^-23
FIELDS = ("n", "sumLo", "sumHi", "sumSq0", "sumSq1", "sumSq2", "mean", "rewardSumSq", "variance", "stdDev", "stdErr")


def w_one() -> np.ndarray:
    """weights under which d1 alone gives fr = d1 exactly (w1 = 1.0)"""
    w = oracle.weights().copy()
    w[1] = 1.0
    return w


def w_one_unit() -> np.ndarray:
    """w_one with w2 = 2^-52: an evaluation with d1 and d2 = 0 present has fr = RN(d1 / (1 + 2^-52))"""
    w = w_one()
    w[2] = 2.0 ** -52
    return w


# ------------------------------------------------------------------------------------------------ the model
def terms(fr: np.ndarray, ok: np.ndarray) -> np.ndarray:
    """rint(fr * 2^52) of the non-null evaluations as int64 (fr * 2^52 is exact, rint rounds half to even as __double2ll_rn)"""
    fr = np.asarray(fr, np.float64)
    return np.rint(np.where(ok, fr, 0.0) * FX).astype(np.int64)[np.asarray(ok, bool)]


def exact_sums(x: np.ndarray) -> tuple[int, int, int]:
    """(n, S1, S2) of int64 terms x as Python ints"""
    xo = np.asarray(x, np.int64).astype(object)
    return int(xo.size), int(xo.sum()) if xo.size else 0, int((xo * xo).sum()) if xo.size else 0


def fields(n: int, s1: int, s2: int) -> dict:
    """one apo_candidate_spread from its integers, with the header's sequence of operations"""
    m = n * s2 - s1 * s1
    assert m >= 0
    mean = math.ldexp(float(s1), -52) / float(n) if n else math.nan
    out = {"n": n, "sumLo": s1 & (2 ** 64 - 1), "sumHi": s1 >> 64, "sumSq0": s2 & (2 ** 64 - 1), "sumSq1": (s2 >> 64) & (2 ** 64 - 1),
           "sumSq2": s2 >> 128, "mean": mean, "rewardSumSq": math.ldexp(float(s2), -104), "S1": s1, "S2": s2, "M": m}
    if n >= 2:
        var = (math.ldexp(float(m), -104) / float(n)) / float(n - 1)
        out.update(variance=var, stdDev=math.sqrt(var), stdErr=math.sqrt(var / float(n)))
    else:
        out.update(variance=math.nan, stdDev=math.nan, stdErr=math.nan)
    return out


def spread_model(fr, ok) -> list[dict]:
    """spreads of rows fr / ok [C][T]"""
    fr, ok = np.atleast_2d(fr), np.atleast_2d(ok)
    return [fields(*exact_sums(terms(fr[c], ok[c]))) for c in range(fr.shape[0])]


def model(dims: np.ndarray, w=None, recip: bool = False) -> list[dict]:
    """spreads of Form D dims [C][T][9] scored whole"""
    return spread_model(*final_rewards(dims, w, recip))


def rec_model(recs: np.ndarray, w=None, recip: bool = False) -> list[dict]:
    return spread_model(*record_final_rewards(recs, w, recip))


def constant_model(n: int, v: float) -> dict:
    """n evaluations at fr = v (v * 2^52 an integer)"""
    x = int(v * FX)
    assert x == v * FX
    return fields(n, n * x, n * x * x)


# ------------------------------------------------------------------------------------------------ fixtures
def const512(T: int = 8192 + 5) -> np.ndarray:
    return np.stack([rows(T, d1=np.float32(-512.0)), rows(T, d1=np.float32(F32_BELOW_512))])


def const2(T: int = 8192 + 5) -> np.ndarray:
    return np.stack([rows(T, d1=np.float32(-F32_BELOW_2)), rows(T, d1=np.float32(F32_BELOW_2))])


def const2_wide() -> np.ndarray:
    """one row of 2^22 + 3 evaluations at -(2 - 2^-23): S2 passes 2^128 over the row"""
    return rows((1 << 22) + 3, d1=np.float32(-F32_BELOW_2))[None]


def one_unit(T: int = 4096 + 33, at: int = 1500) -> np.ndarray:
    """[1][T][9] under w_one_unit: d1 = 1.5 everywhere, d2 = 0 present at one position only"""
    d = rows(T, d1=np.float32(1.5))
    d[at, 2] = 0.0
    return d[None]


def _rn_cases():
    """(name, m, p, q) for the four RN(M) edges, M = p q m^2.  m is odd, so m^2 = 1 mod 8 and the three low bits of M are
    those of p q; m only sets M's bit length"""
    want = {                                    # bit length of M, (p, q), three low bits (significand LSB | round | sticky)
        "tie_even_down": (54, (127, 131), lambda v: (v & 3) == 1),     # ...0|1: a tie, the kept significand is even
        "tie_up": (54, (127, 129), lambda v: (v & 3) == 3),            # ...1|1: a tie, the kept significand is odd
        "sticky_above": (55, (125, 127), lambda v: (v & 7) == 3),      # ...0|1|1: half an ulp and a sticky bit: up, though even
        "below_half": (55, (127, 131), lambda v: (v & 7) == 5),        # ...1|0|1: below half an ulp: down, though odd
    }
    out = []
    for name, (bits, (p, q), ok) in want.items():
        r = p * q
        m = math.isqrt((1 << (bits - 1)) // r) | 1                       # the smallest odd m near the bit length
        while (r * m * m).bit_length() < bits:
            m += 2
        assert (r * m * m).bit_length() == bits and ok(r * m * m) and m < 1 << 24
        out.append((name, m, p, q))
    return out


RN_CASES = _rn_cases()
RN_T = 260


def rn_edges() -> np.ndarray:
    """[4][RN_T][9]: row k holds p evaluations at d1 = m 2^-52 and q at d1 = 0, interleaved, then null ones (m < 2^24: an fp32)"""
    out = []
    for _, m, p, q in RN_CASES:
        v = np.float32(m * 2.0 ** -52)
        assert float(v) * FX == m
        r = rows(RN_T, d1=np.float32(0))
        r[p + q:, 1] = NAN
        r[np.arange(p) * 2, 1] = v
        out.append(r)
    return np.stack(out)


def counts(T: int = 2 * 1024 + 33) -> np.ndarray:
    """[6][T][9]: 0, 1 and 2 non-null evaluations; every third null; alternating +-1 (even and odd n)"""
    d = np.full((6, T, 9), NAN, np.float32)
    d[1, 700, 1] = 0.25
    d[2, 5, 1], d[2, T - 1, 1] = -0.5, 0.375
    g = oracle.gen_dims(0x5EED7001, 0, 1, 0, T, 300, 4)[0]
    d[3] = g
    d[3, ::3] = NAN
    d[4, :, 1] = np.where(np.arange(T) % 2 == 0, 1.0, -1.0)
    d[5, :T - 1, 1] = np.where(np.arange(T - 1) % 2 == 0, 1.0, -1.0)
    return d


def tails(seed: int = 3):
    """one [2][T][9] generator tensor per T = 1024 + r, r in TAILS"""
    return [oracle.gen_dims(0x5EED7100 + seed, 0, 2, 0, 1024 + r, 300, 4) for r in TAILS]


def all_fixtures():
    """(name, dims, w) of every fixture above but const2_wide; const512 only on the routes whose domain admits it"""
    out = [("const512", const512(), w_one()), ("const2", const2(), w_one()), ("one_unit", one_unit(), w_one_unit()),
           ("rn_edges", rn_edges(), w_one()), ("counts", counts(), w_one())]
    out += [(f"tail_{d.shape[1]}", d, None) for d in tails()]
    return out
