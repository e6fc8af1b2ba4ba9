"""Corpora built to reach the flush points and the example merges of the corpus scan (csrc/apo_corpus.cuh scan_record /
scan_flush, in every host that runs them) and of the per-candidate passes (csrc/apo_cand.cu).

Two kinds of data, both built from a small table of distinct records indexed by a uint8 array, so a 36 M-record corpus costs
its own 1.15 GB and little more:

- saturating(): every record identical -- 'bad', one mode, one category in every packed counter, a chosen subset of the six
  pattern predicates.  Every lane of every host fills the same packed fields to the flush cadence, and the report has a closed
  form (closed_form), computed here in exact integers.
- planted(): a background that hits no pattern ('good' / none records and a few 'bad' records that match no predicate), with
  hits of each pattern planted at chosen positions (SCENARIOS): the earliest hit late in the range, pairs on both sides of
  block boundaries, crowded 32-record groups, a dense tail.  Returns the records with the designed pattern counts and first
  three examples.

Plain helpers, imported by the tests that use them (no fixtures, no GPU)."""
import numpy as np

import oracle

F_ERRORS, F_ENDED, F_VALID, F_FAILSPAN = 0x01, 0x02, 0x08, 0x10
FX = 1 << 52
BLOCKS = (32, 1024, 2048, 8192, 131072)        # warp group, cand tile, K2 tile, K1t tile, a large power of two
MINC = (2, 2, 3, 2, 2, 2)                      # APO:645,671,695,715,736,756


def _rec(**kw):
    r = np.zeros(1, oracle.RECORD_DTYPE)
    base = dict(feedback=1, flags=F_VALID | F_ENDED, mode=1, userMsgs=1, asstMsgs=1, toolCalls=1, toolSucc=1, toolFail=0,
                llmCalls=1, tokens=500, toolDurMs=100.0)
    base.update(kw)
    for k, v in base.items():
        r[k] = v
    return r


def hit_record(preds, mode=1, feedback=2):
    """a record carrying the predicates `preds` (subset of 0..5) and no other; 'bad' unless told otherwise"""
    s = set(preds)
    return _rec(feedback=feedback, mode=mode,
                flags=F_VALID | F_ENDED | (F_ERRORS if 0 in s else 0) | (F_FAILSPAN if 1 in s else 0),
                toolCalls=4, toolFail=1 if 1 in s else 0, toolSucc=3 if 1 in s else 4,
                tokens=10_001 if 2 in s else 1_500, llmCalls=3 if 3 in s else 2, userMsgs=4 if 4 in s else 2, asstMsgs=3,
                toolDurMs=4 * 20_000.0 if 5 in s else 4 * 2_000.0)


# ------------------------------------------------------------------------------------------------ saturating corpora
def saturating(T, preds, mode=1, row=32):
    """T identical 'bad' records in `mode` with the predicates `preds`.  row=16: Form R16 (numpy, no record copy per row)."""
    rec = hit_record(preds, mode)
    if row == 16:
        rec = oracle_pack16(rec)
    return np.broadcast_to(rec, (T,)).copy()


def closed_form(T, preds, mode=1, idx_base=0):
    """The report of saturating(T, preds, mode) as exact integers (sums as 2^-52 fixed point) plus the derived fields."""
    rec = hit_record(preds, mode)
    d, m = oracle.reward_dims(rec)
    _, _, fr = oracle.reward_one(rec)
    dims = []
    for i in range(oracle.NDIM):
        present = (m >> i) & 1
        fx = T * int(np.rint(d[i] * FX)) if present else 0
        n = T if present else 0
        s = float(fx) / FX
        avg = s / n if n else 0.0
        dims.append({"fx": fx, "sum": s, "count": n, "avg": avg,
                     "low_flag": int(n >= 5 and avg < -0.3), "sugg_flag": int(n >= 3 and avg < 0.0)})
    rfx = T * int(np.rint(fr * FX))
    by_mode = [[0, 0, 0] for _ in range(oracle.NMODE)]
    by_mode[mode] = [T, 0, T]
    s = set(preds)
    pats = [{"count": T if p in s else 0, "flag": int(p in s and T >= MINC[p]),
             "examples": [idx_base + k if (p in s and k < T) else -1 for k in range(3)]} for p in range(oracle.NPAT)]
    tc, ts, tf = (int(rec[f][0]) for f in ("toolCalls", "toolSucc", "toolFail"))
    return {"total": T, "good": 0, "bad": T, "none": 0, "byMode": by_mode, "withReward": T, "rewardFx": rfx,
            "rewardSum": float(rfx) / FX, "avgReward": (float(rfx) / FX) / T, "dim": dims, "pat": pats,
            "toolCalls": T * tc, "toolSucc": T * ts, "toolFail": T * tf}


def check_closed_form(rep, want):
    """every integer of `want` exactly; every binary64 field bit for bit (the engine sums exactly and rounds once)"""
    assert (rep.total, rep.good, rep.bad, rep.none) == (want["total"], want["good"], want["bad"], want["none"])
    assert rep.goodRate == 0.0
    for m in range(oracle.NMODE):
        assert list(rep.byMode[m]) == want["byMode"][m], m
    assert rep.withReward == want["withReward"]
    assert rep.rewardSum == want["rewardSum"] and rep.avgReward == want["avgReward"]
    for i, w in enumerate(want["dim"]):
        assert (rep.dim[i].count, rep.dim[i].sum, rep.dim[i].avg) == (w["count"], w["sum"], w["avg"]), i
        assert (rep.dim[i].low_flag, rep.dim[i].sugg_flag) == (w["low_flag"], w["sugg_flag"]), i
    for p, w in enumerate(want["pat"]):
        assert (rep.pat[p].count, rep.pat[p].flag, list(rep.pat[p].examples)) == (w["count"], w["flag"], w["examples"]), p
    assert (rep.toolCalls, rep.toolSucc, rep.toolFail) == (want["toolCalls"], want["toolSucc"], want["toolFail"])


# ------------------------------------------------------------------------------------------------ planted corpora
def scenario_positions(kind, T, shift=0):
    """positions of one pattern's hits in [0, T) for scenario `kind`; `shift` moves the late positions to sweep boundaries"""
    late = T - 1 - shift
    if kind == 0:                                  # earliest hit in the last 2048-record tile
        pos = [late - 2000, late - 700, late]
    elif kind == 1:                                # the last lane of a 32-record group, then the last record
        g = (T // 2 + shift) // 32
        pos = [g * 32 + 31, T - 1]
    elif kind == 2:                                # pairs at k*B - 1 and k*B for every block size B
        pos = []
        for B in BLOCKS:
            k = max(1, (T - shift) // B - 1) if B < T else 0
            if k:
                pos += [k * B - 1, k * B]
    elif kind == 3:                                # > 3 hits in one 32-record group, one earlier hit in another warp's range
        g = (T - 4096 - shift) // 32
        pos = [T // 3 + 17 + shift] + [g * 32 + o for o in (0, 5, 9, 20, 31)]
    elif kind == 4:                                # a dense block at the end plus a single earlier hit
        pos = [T // 5 + 3 + shift] + list(range(T - 600, T))
    else:                                          # only the last three records
        pos = [T - 3 - shift, T - 2 - shift, T - 1 - shift]
    return sorted({p for p in pos if 0 <= p < T})


def plant_plan(T, kinds=range(6), shift=0, extra=None):
    """{pattern: sorted positions}: pattern p gets scenario kinds[p]; extra = {pattern: more positions}"""
    plan = {p: scenario_positions(k, T, shift) for p, k in zip(range(oracle.NPAT), kinds)}
    for p, more in (extra or {}).items():
        plan[p] = sorted(set(plan[p]) | {q for q in more if 0 <= q < T})
    return plan


def table(row=32):
    """the distinct records: 0-4 good (mode 0-4), 5-9 none, 10-14 'bad' hitting nothing, 15 + mask 'bad' hitting the patterns
    of the 6-bit mask (mask 1-63; a record where two plans meet carries both predicates)"""
    recs = [_rec(mode=m) for m in range(5)] + [_rec(feedback=0, mode=m) for m in range(5)]
    recs += [_rec(feedback=2, mode=m) for m in range(5)]
    recs += [hit_record([p for p in range(oracle.NPAT) if (mask >> p) & 1]) for mask in range(1, 64)]
    t = np.concatenate(recs)
    return oracle_pack16(t) if row == 16 else t


def background_index(T):
    """per record: kind * 5 + mode; mostly good, every 7th none, every 4099th a 'bad' record that hits nothing"""
    t = np.arange(T, dtype=np.uint32)
    idx = (t % 5).astype(np.uint8)
    idx[t % 7 == 3] += 5
    idx[t % 4099 == 11] = 10 + idx[t % 4099 == 11] % 5
    return idx


def planted(T, kinds=range(6), shift=0, extra=None, row=32, idx_base=0):
    """(records, plan, designed): the background with the plan's hits; designed = per pattern (count, first three examples
    as absolute positions, -1 padded) and the number of 'bad' records"""
    plan = plant_plan(T, kinds, shift, extra)
    idx = background_index(T)
    mask = np.zeros(T, np.uint8)
    for p, pos in plan.items():
        mask[np.asarray(pos, np.int64)] |= np.uint8(1 << p)
    hit = mask != 0
    idx[hit] = 14 + mask[hit]
    recs = table(row)[idx]
    return recs, plan, designed(idx, plan, idx_base)


def designed(idx, plan, idx_base=0):
    bad = int(np.count_nonzero((idx >= 10)))
    pats = [(len(plan[p]), [idx_base + q for q in plan[p][:3]] + [-1] * (3 - min(3, len(plan[p])))) for p in range(oracle.NPAT)]
    return {"bad": bad, "pat": pats, "badExamples": [idx_base + int(q) for q in np.flatnonzero(idx >= 10)[:3]]}


def check_designed(rep, want):
    assert rep.bad == want["bad"]
    for p, (n, ex) in enumerate(want["pat"]):
        assert (rep.pat[p].count, list(rep.pat[p].examples)) == (n, ex), p


def oracle_pack16(recs):
    """Form R -> Form R16 with the engine's packing rule (apo_format.h pack16), in numpy: the tests need it without a GPU"""
    recs = np.ascontiguousarray(recs, oracle.RECORD_DTYPE)
    assert np.all(recs["toolSucc"] + recs["toolFail"] == recs["toolCalls"]) and np.all(recs["toolCalls"] <= 65535)
    out = np.zeros(recs.shape, oracle.RECORD16_DTYPE)
    f = recs["flags"]
    out["hdr"] = ((recs["feedback"] & 3) | np.where(f & F_ERRORS, 4, 0) | np.where(f & F_ENDED, 8, 0) | np.where(f & F_VALID, 16, 0)
                  | np.where(f & F_FAILSPAN, 32, 0) | ((recs["mode"].astype(np.uint16) & 7) << 6)).astype(np.uint16)
    out["userMsgs"] = np.minimum(recs["userMsgs"], 255)
    out["asstMsgs"] = np.minimum(recs["asstMsgs"], 255)
    out["toolCalls"] = recs["toolCalls"]
    out["toolFail"] = recs["toolFail"]
    out["llmCalls"] = np.minimum(recs["llmCalls"], 255)
    out["durClass"] = recs["durClass"]
    out["tokens"] = np.minimum(recs["tokens"], 65535)
    out["toolDurMs"] = recs["toolDurMs"]
    return out


# ------------------------------------------------------------------------------------------------ sparse 'bad' evaluations
def sparse_bad_dims(dims, positions):
    """Form D rows whose only 'bad' evaluations (d0 = -1) are `positions[c]` of row c: every other -1 becomes 1"""
    d0 = dims[:, :, 0]
    d0[d0 == -1.0] = 1.0
    for c, pos in enumerate(positions):
        d0[c, np.asarray(pos, np.int64)] = -1.0
    return dims


def sparse_bad_positions(C, T, tile=1024, seed=0):
    """per row a few 'bad' positions, all late: the last tile, the last lane of a 32-record group, both sides of a tile boundary,
    a crowded group; rows rotate through the scenarios and shift them, and some rows get fewer than three"""
    out = []
    for c in range(C):
        k = c % 5
        s = 96 * (c // 5)
        if k == 0:
            pos = [T - 1 - s]
        elif k == 1:
            pos = [((T - tile - s) // 32) * 32 + 31, T - 1]
        elif k == 2:
            b = ((T - s) // tile - 1) * tile
            pos = [b - 1, b]
        elif k == 3:
            g = ((T - 3 * tile - s) // 32) * 32
            pos = [g + o for o in (0, 3, 7, 31)]
        else:
            pos = [T // 2 + 5 + s, T - 2, T - 1]
        out.append(sorted({p for p in pos if 0 <= p < T}))
    return out
