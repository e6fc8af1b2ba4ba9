"""Label planes and Form D tensors that reach the edges of the per-candidate group scores (csrc/apo_cand.cu k_cand_groups /
k_cand_groups_report), and two models of the scores they are checked against.

A candidate's score in group g covers its evaluations on the records t with labels[t] == g: the feedback tallies, the
number of non-null evaluations and the exact integer sum of rint(fr * 2^52), rounded once to binary64 (rewardSum) and
divided by that number (avgReward, NaN when it is 0).  fr is extremes_fixtures.final_rewards /
record_final_rewards, the scoring arithmetic restated in numpy.  group_model sums every group's terms as Python ints;
group_model_split adds the low and high 32-bit halves of the terms with np.add.at instead, the way the limbs are kept on
the device.  The CPU tests check that both agree on every fixture and that the groups of a candidate add up to its
scoring integers; the GPU tests compare the engine with group_model bit for bit.

- zero: every label 0 (G = 1), where every field equals the breakdown's.
- mod: labels t % G for G = 2, 5 and 64, a new label on every record.
- edges: runs that change label at lane 31 / 32 of a group of 32 and at the 1024-record edges of a warp tile.
- last: a group present only at the last record, T = 1024 k + r for r in TAILS, and a group with no record at all.
- wide: d0 = +-511 alone over 2^20 records, so each group's sum passes 2^64, cancelling between the two groups of c0.
- null: a group whose records are all null (withReward 0, avgReward NaN) while its tallies still count.

Plain helpers (no pytest fixtures, no GPU)."""
from __future__ import annotations

import math

import numpy as np

import oracle
from extremes_fixtures import NAN, final_rewards, record_final_rewards, rows

TAILS = (1, 31, 33, 1023)
FX = float(2 ** 52)


def dims_tally(dims: np.ndarray) -> np.ndarray:
    """tally of Form D / Q / P / T evaluations from d0 (TCS:677-679): 1 good, 2 bad, 0 none"""
    d0 = np.asarray(dims)[..., 0].astype(np.float64)
    return np.where(d0 == 1.0, 1, np.where(d0 == -1.0, 2, 0))


def record_tally(recs: np.ndarray) -> np.ndarray:
    """tally of Form R / R16 records from the feedback field, VALID or not"""
    fb = np.asarray(recs)["feedback"]
    return np.where(fb == 1, 1, np.where(fb == 2, 2, 0))


def terms(fr: np.ndarray) -> np.ndarray:
    """rint(fr * 2^52) as int64 (fr * 2^52 is exact, rint rounds half to even as __double2ll_rn)"""
    return np.rint(np.asarray(fr) * FX).astype(np.int64)


def score_of(total: int, good: int, bad: int, n: int, s: int) -> dict:
    """one apo_group_score from the integers: the report rules of the breakdown"""
    rsum = float(s) / FX                        # int -> binary64 rounds once, scaling by 2^-52 is exact
    return {"total": total, "good": good, "bad": bad, "goodRate": good / (good + bad) if good + bad else 0.0,
            "withReward": n, "rewardSum": rsum, "avgReward": rsum / n if n else math.nan, "sum": s}


def group_model(fr, ok, tally, labels, G: int) -> list[list[dict]]:
    """[C][G] scores of rows fr / ok / tally [C][T] whose record t has labels[t]; sums as Python ints"""
    fr, ok, tally, labels = np.atleast_2d(fr), np.atleast_2d(ok), np.atleast_2d(tally), np.asarray(labels)
    fx = np.where(ok, terms(np.where(ok, fr, 0.0)), 0)
    out = []
    for c in range(fr.shape[0]):
        row = []
        for g in range(G):
            m = labels == g
            row.append(score_of(int(m.sum()), int((tally[c][m] == 1).sum()), int((tally[c][m] == 2).sum()), int(ok[c][m].sum()),
                                int(fx[c][m].astype(object).sum())))
        out.append(row)
    return out


def group_model_split(fr, ok, tally, labels, G: int) -> list[list[dict]]:
    """the same scores from the low and high 32-bit halves of every term, added per group with np.add.at"""
    fr, ok, tally, labels = np.atleast_2d(fr), np.atleast_2d(ok), np.atleast_2d(tally), np.asarray(labels, np.int64)
    fx = np.where(ok, terms(np.where(ok, fr, 0.0)), 0)
    C = fr.shape[0]
    lo, hi = np.zeros((C, G), np.int64), np.zeros((C, G), np.int64)
    cnt = np.zeros((C, 5, G), np.int64)
    for c in range(C):
        np.add.at(lo[c], labels, fx[c] & 0xFFFFFFFF)
        np.add.at(hi[c], labels, fx[c] >> 32)
        for k, v in enumerate((np.ones_like(labels), tally[c] == 1, tally[c] == 2, ok[c])):
            np.add.at(cnt[c, k], labels, v.astype(np.int64))
    return [[score_of(int(cnt[c, 0, g]), int(cnt[c, 1, g]), int(cnt[c, 2, g]), int(cnt[c, 3, g]), (int(hi[c, g]) << 32) + int(lo[c, g]))
             for g in range(G)] for c in range(C)]


def model(dims: np.ndarray, labels, G: int, w=None, recip: bool = False) -> list[list[dict]]:
    """scores of Form D dims [C][T][9] scored whole; labels [T] of the same positions"""
    fr, ok = final_rewards(dims, w, recip)
    return group_model(fr, ok, dims_tally(dims), labels, G)


def rec_model(recs: np.ndarray, labels, G: int, w=None, recip: bool = False) -> list[list[dict]]:
    fr, ok = record_final_rewards(recs, w, recip)
    return group_model(fr, ok, record_tally(recs), labels, G)


# ------------------------------------------------------------------------------------------------ fixtures
def gen(seed: int, C: int, T: int) -> np.ndarray:
    return oracle.gen_dims(0x5EED6000 + seed, 0, C, 0, T, 300, 4)


def zero():
    T = 3 * 1024 + 77
    return gen(1, 3, T), np.zeros(T, np.uint8), 1


def mod(G: int):
    T = 4 * 1024 + 5
    return gen(2, 2, T), (np.arange(T) % G).astype(np.uint8), G


def edges():
    """G = 4: twice the tile index (t // 1024), bumped by one at lane 31 of every group of 32, mod 4"""
    T = 5 * 1024 + 40
    t = np.arange(T)
    return gen(3, 2, T), ((2 * (t // 1024) + (t % 32 == 31)) % 4).astype(np.uint8), 4


def last(r: int):
    """G = 3: group 1 only at the last record, group 2 nowhere"""
    T = 1024 + r
    labels = np.zeros(T, np.uint8)
    labels[-1] = 1
    return gen(4 + r, 2, T), labels, 3


WIDE_T = 1 << 20


def wide():
    """[2][2^20][9], d0 alone, G = 2 (group 1 = the second half): c0 = +511 on group 0 and -511 on group 1, whose sums of
    about +-2^80 cancel in the candidate's; c1 = -511 everywhere"""
    T = WIDE_T
    d = np.repeat(rows(T, d0=np.float32(511.0))[None], 2, axis=0)
    d[0, T // 2:, 0] = -511.0
    d[1, :, 0] = -511.0
    return d, (np.arange(T) >= T // 2).astype(np.uint8), 2


def null():
    """G = 3: the records of group 1 are all null under W_NULL (only d0 and d3 present, which carry no weight), while d0
    still gives them tallies"""
    T = 2 * 1024 + 9
    d = gen(5, 2, T)
    labels = (np.arange(T) % 3).astype(np.uint8)
    d[:, labels == 1, :] = NAN
    d[:, labels == 1, 0] = np.where(np.arange(int((labels == 1).sum())) % 2 == 0, 1.0, -1.0)
    d[:, labels == 1, 3] = 0.5
    return d, labels, 3


W_NULL = np.array([0.0, 0.18, 0.12, 0.0, 0.05, 0.05, 0.08, 0.08, 0.11])   # d0 and d3 carry no weight


def all_fixtures():
    """(name, dims, labels, G, w) of every fixture above but wide, which weighs d0 alone and is 2^20 records long"""
    out = [("zero",) + zero() + (None,)]
    out += [(f"mod{G}",) + mod(G) + (None,) for G in (2, 5, 64)]
    out += [("edges",) + edges() + (None,)]
    out += [(f"last_{1024 + r}",) + last(r) + (None,) for r in TAILS]
    out += [("null",) + null() + (W_NULL,)]
    return out


def w_d0() -> np.ndarray:
    """weights under which d0 alone carries a reward (the wide fixture)"""
    w = oracle.weights().copy()
    if w[0] == 0.0:
        w[0] = 1.0
    return w
