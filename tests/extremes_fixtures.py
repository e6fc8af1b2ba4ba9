"""Hand-built Form D tensors that reach the edges of the per-candidate extremes (csrc/apo_cand.cu k_cand_extremes /
k_cand_extremes_merge), and two models of the lists they are checked against.

A candidate's lists hold, over its evaluations with a non-null finalReward, the 32 lowest (finalReward ascending) and the
32 highest (finalReward descending), ties -> lower record position.  final_rewards restates the scoring arithmetic per
evaluation in numpy (binary64, no FMA, the push order of tests/k1_fixtures.fx_model, ws * RN(1/tw) with recip);
extremes_sorted takes the lists from one numpy lexsort over (finalReward, position); extremes_inserted builds them by
inserting every evaluation into two sorted 32-slot arrays, in position order.  The CPU tests check that both agree on every
fixture; the GPU tests compare the engine with them bit for bit.

- ties: every reward equal, so the lists are the first 32 positions.
- counts: rows with 0, 1, 31, 32 and 33 non-null evaluations among null ones.
- null rows: only dimensions of weight 0 present (total weight 0), under custom weights.
- ulps: fp32 values one ulp apart, interleaved, so neighbouring rewards differ in the last bits.
- falling: a strictly falling row, the worst case of the per-warp merge (every group of 32 enters the lowest list).
- last: the minimum at the last position and the maximum just before it.
- tails: rows of T = 1024 k + r, r in {1, 31, 32, 33, 1023}, so the last warp tile of a row is nearly empty or nearly full.

Plain helpers (no pytest fixtures, no GPU)."""
from __future__ import annotations

import numpy as np

import oracle

N = 32
NAN = np.float32("nan")
TAILS = (1, 31, 32, 33, 1023)
W_ZERO = np.array([0.0, 1.0, 0.5, 0.0, 0.25, 0.0, 0.125, 0.0625, 0.0])   # d0, d3, d5, d8 carry no weight


def final_rewards(dims: np.ndarray, w=None, recip: bool = False):
    """(fr, ok) of dims [..., T, 9] (fp32 or binary64, NaN = absent): finalReward per evaluation, +0.0 for a zero, and
    whether it is non-null (total weight of the present dimensions > 0)"""
    w = oracle.weights() if w is None else np.asarray(w, np.float64)
    d = np.asarray(dims).astype(np.float64)
    p = ~np.isnan(d)
    g = np.where(p, d, 0.0)
    ws = np.zeros(d.shape[:-1])
    tw = np.zeros(d.shape[:-1])
    for i in range(9):
        ws = ws + g[..., i] * w[i]
        tw = tw + np.where(p[..., i], w[i], 0.0)
    ok = tw > 0
    with np.errstate(divide="ignore", invalid="ignore"):
        fr = ws * (1.0 / tw) if recip else ws / tw
    fr = np.where(ok, fr, 0.0) + 0.0                     # -0.0 + 0.0 == +0.0
    return fr, ok


def record_final_rewards(recs: np.ndarray, w=None, recip: bool = False):
    """(fr, ok) of Form R records [..., T]: the oracle's dimensions (TCS:668-763), the VALID flag, then final_rewards"""
    recs = np.asarray(recs)
    flat = recs.reshape(-1)
    dims = np.full((flat.size, 9), np.nan)
    for i, r in enumerate(flat):
        d, m = oracle.reward_dims(r)
        dims[i] = np.where([(m >> k) & 1 for k in range(9)], d, np.nan)
    fr, ok = final_rewards(dims, w, recip)
    ok &= (flat["flags"] & 0x08) != 0
    return fr.reshape(recs.shape), ok.reshape(recs.shape)


def _lists(n, lo_pos, lo_fr, hi_pos, hi_fr):
    out = {"n": n, "lowest": [-1] * N, "lowestReward": [float("nan")] * N, "highest": [-1] * N, "highestReward": [float("nan")] * N}
    out["lowest"][:n], out["lowestReward"][:n] = [int(x) for x in lo_pos], [float(x) for x in lo_fr]
    out["highest"][:n], out["highestReward"][:n] = [int(x) for x in hi_pos], [float(x) for x in hi_fr]
    return out


def extremes_sorted(fr: np.ndarray, ok: np.ndarray, positions) -> dict:
    """the lists of one row by a lexsort over (finalReward, position); positions: the record position of every evaluation"""
    pos = np.asarray(positions, np.int64)[ok]
    v = np.asarray(fr)[ok]
    lo = np.lexsort((pos, v))[:N]
    hi = np.lexsort((pos, -v))[:N]
    return _lists(min(N, v.size), pos[lo], v[lo], pos[hi], v[hi])


def extremes_inserted(fr: np.ndarray, ok: np.ndarray, positions) -> dict:
    """the same lists by inserting each evaluation, in the order given, into two sorted arrays of at most 32 slots"""
    low, high = [], []                                   # (key, position, reward)
    for f, k, p in zip(np.asarray(fr).tolist(), np.asarray(ok).tolist(), np.asarray(positions).tolist()):
        if not k:
            continue
        for lst, key in ((low, (f, p)), (high, (-f, p))):
            if len(lst) == N and not key < lst[-1][0]:
                continue
            i = len(lst)
            while i > 0 and key < lst[i - 1][0]:
                i -= 1
            lst.insert(i, (key, p, f))
            del lst[N:]
    return _lists(len(low), [e[1] for e in low], [e[2] for e in low], [e[1] for e in high], [e[2] for e in high])


def model(dims: np.ndarray, w=None, recip: bool = False, idx_base: int = 0) -> list[dict]:
    """the lists of every row of Form D dims [C][T][9] scored whole (positions idx_base + t)"""
    fr, ok = final_rewards(dims, w, recip)
    return [extremes_sorted(fr[c], ok[c], idx_base + np.arange(fr.shape[1])) for c in range(fr.shape[0])]


# ------------------------------------------------------------------------------------------------ fixtures
def rows(n: int, **dims) -> np.ndarray:
    """n evaluations with dimension i = dims[f'd{i}'] (scalar or array), every other dimension absent"""
    r = np.full((n, 9), NAN, np.float32)
    for k, v in dims.items():
        r[:, int(k[1:])] = v
    return r


def ties(T: int = 1024 + 77) -> np.ndarray:
    """[2][T][9]: every reward equal (all d1 = 0.5; then d1 = 0.5 and d2 = -0.25 everywhere)"""
    return np.stack([rows(T, d1=0.5), rows(T, d1=0.5, d2=-0.25)])


def counts(T: int = 2 * 1024 + 33) -> np.ndarray:
    """[5][T][9]: 0, 1, 31, 32 and 33 non-null evaluations spread over the row, the rest all-NaN (null)"""
    d = np.full((5, T, 9), NAN, np.float32)
    rng = np.random.default_rng(5)
    for c, n in enumerate((0, 1, 31, 32, 33)):
        at = np.sort(rng.choice(T, n, replace=False))
        d[c, at, 1] = rng.integers(-8, 8, n).astype(np.float32) / 8   # ties among them too
        d[c, at, 2] = rng.integers(-4, 4, n).astype(np.float32) / 4
    return d


def null_rows(T: int = 1024 + 40) -> np.ndarray:
    """[3][T][9] for W_ZERO: c0 only zero-weight dimensions (every evaluation null), c1 half null, c2 null but d0 present"""
    d = np.repeat(rows(T, d0=1.0, d3=-0.5, d8=0.3)[None], 3, axis=0)
    d[1, ::2, 1] = np.linspace(-1, 1, (T + 1) // 2, dtype=np.float32)
    d[2, :, 5] = -1.0
    return d


def ulps(T: int = 1024 + 96) -> np.ndarray:
    """[2][T][9]: d1 = +-0.37 and its fp32 neighbours, 8 of each at random positions (c0) or in runs (c1), among d1 = 0, so
    each list steps through three rewards one fp32 ulp apart before it reaches the zeros"""
    base = np.float32(0.37)
    v = np.array([base, np.nextafter(base, np.float32(1)), np.nextafter(base, np.float32(-1)),
                  -base, np.nextafter(-base, np.float32(1)), np.nextafter(-base, np.float32(-1))], np.float32)
    a = np.zeros(T, np.float32)
    b = np.zeros(T, np.float32)
    a[np.random.default_rng(7).choice(T, 48, replace=False)] = np.repeat(v, 8)
    b[T // 2:T // 2 + 48] = np.repeat(v, 8)
    return np.stack([rows(T, d1=a), rows(T, d1=b)])


def falling(T: int = 3 * 1024 + 5, C: int = 1) -> np.ndarray:
    """[C][T][9]: d1 strictly falling along the row (distinct fp32 values), so every group of 32 enters the lowest list"""
    v = np.float32(1) - np.arange(T, dtype=np.float64) * (1.0 / 2 ** 23)
    assert np.all(np.diff(v.astype(np.float32)) < 0)
    return np.repeat(rows(T, d1=v.astype(np.float32))[None], C, axis=0)


def last(T: int = 2 * 1024 + 31) -> np.ndarray:
    """[1][T][9]: the maximum at T - 2 and the minimum at T - 1, every other reward in between"""
    d = rows(T, d1=np.float32(0.25))
    d[T - 2, 1], d[T - 1, 1] = 0.75, -0.75
    return d[None]


def tails(seed: int = 3):
    """one [2][T][9] tensor per T = 1024 k + r, r in TAILS (k = 0, 1): categorical generator rows"""
    return [oracle.gen_dims(0x5EED2000 + seed, 0, 2, 0, T, 300, 4) for r in TAILS for T in (r, 1024 + r)]


def all_fixtures():
    """(name, dims, w) of every fixture above"""
    out = [("ties", ties(), None), ("counts", counts(), None), ("null_rows", null_rows(), W_ZERO), ("ulps", ulps(), None),
           ("falling", falling(), None), ("last", last(), None)]
    out += [(f"tail_{d.shape[1]}", d, None) for d in tails()]
    return out
