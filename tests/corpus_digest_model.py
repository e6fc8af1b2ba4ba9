"""numpy model of the corpus digest (csrc/apo_kernels.h CorpusDigestParams, built at a corpus load by build_digest).

A VALID record reaches the weight-dependent words of the corpus report (finalReward sum, withReward, per-dimension census)
only through its reward key: the (feedback, hasErrors, endTime) slot i01 = fb + 3 err + 6 ended, the level of d3..d8 (the
last slot of a group = not pushed: 4, d6: 6) and the binary64 bit pattern of d2 (+0.0 when not pushed).  The digest holds
each distinct key once with its record count, packed as {d2 bits, slots | count << 22}; and the 45 words no weight reaches:
tallies, byMode, pattern counts, tool totals (the corpus block's words CORP_TALLY..CORP_NREC) and the first three 'bad'
records of each pattern as inverted indices."""
from collections import Counter

import numpy as np

COUNT_SHIFT = 22
SHIFTS = (0, 4, 7, 10, 13, 16, 19)                      # i01, i3, i4, i5, i6, i7, i8
ABSENT = {3: 4, 4: 4, 5: 4, 6: 6, 7: 4, 8: 4}
LEVELS = {3: (1.0, -0.2, -0.5, -1.0), 4: (1.0, 0.3, -0.3, -0.8), 5: (1.0, 0.5, 0.0, -0.5), 7: (1.0, 0.5, 0.0, -0.5),
          8: (1.0, 0.3, -0.3, -0.8)}
LEVELS[6] = tuple(max(-1.0, 1.0 - k * 0.4) for k in range(6))           # TCS:735


def _u(a):
    return np.asarray(a).astype(np.uint64)


def keys(recs):
    """(d2 bits uint64, slots uint64, valid bool) per record, by the index rules of record_ws_table_t"""
    r = np.asarray(recs).reshape(-1)
    fb = r["feedback"].astype(np.int64)
    fb = np.where(fb < 3, fb, 0)
    err = (r["flags"] & 1).astype(np.int64)
    ended = ((r["flags"] >> 1) & 1).astype(np.int64)
    agent = r["mode"] == 2
    tc = r["toolCalls"].astype(np.int64)
    tool = tc > 0
    total = np.where(tool, tc, 1).astype(np.float64)
    rate = r["toolSucc"].astype(np.float64) / total
    d2 = np.where(tool, rate * 2.0 - 1.0, 0.0)
    tf = r["toolFail"].astype(np.int64)
    i3 = (tf >= np.where(agent, 2, 1)).astype(np.int64) + (tf >= np.where(agent, 3, 2)) + (tf >= np.where(agent, 5, 3))
    i4 = (tc > np.where(agent, 8, 3)).astype(np.int64) + (tc > np.where(agent, 15, 6)) + (tc > np.where(agent, 25, 10))
    dc = r["durClass"].astype(np.int64)
    dur = r["toolDurMs"].astype(np.float64)
    derived_level = (dur > 1000.0 * total).astype(np.int64) + (dur > 3000.0 * total) + (dur > 10000.0 * total)
    level = np.where(dc & 0x80, dc & 3, derived_level)
    pos = np.where(dc & 0x80, (dc & 4) != 0, dur > 0.0)
    llm = r["llmCalls"].astype(np.int64)
    over = np.maximum(llm - np.where(agent, 3, 1), 0)
    tok = r["tokens"].astype(np.int64)
    i7 = (tok > np.where(agent, 5000, 2000)).astype(np.int64) + (tok > np.where(agent, 15000, 5000)) + (tok > np.where(agent, 30000, 10000))
    turns = np.minimum(r["userMsgs"].astype(np.int64), r["asstMsgs"].astype(np.int64))
    thr = np.where(agent, 3, 2)
    i8 = (turns > thr).astype(np.int64) + (turns > 2 * thr) + (turns > 3 * thr)
    idx = (fb + 3 * err + 6 * ended,
           np.where(tool, i3, 4), np.where(tool, i4, 4), np.where(tool & pos, level, 4),
           np.where(llm > 0, np.minimum(over, 5), 6), np.where(tok > 0, i7, 4), np.where(turns > 0, i8, 4))
    slots = np.zeros(len(r), np.uint64)
    for v, s in zip(idx, SHIFTS):
        slots |= _u(v) << np.uint64(s)
    return d2.view(np.uint64), slots, (r["flags"] & 0x08) != 0


def digest(recs):
    """{(d2 bits, slots): count} over the VALID records"""
    d2, s, v = keys(recs)
    return Counter(zip(d2[v].tolist(), s[v].tolist()))


def entries(recs):
    """the digest as the device packs it, sorted"""
    return sorted((d, s | (n << COUNT_SHIFT)) for (d, s), n in digest(recs).items())


def unpack(slots):
    return [(int(slots) >> s) & (15 if s == 0 else 7) for s in SHIFTS]


def key_dims(d2bits, slots):
    """the nine dimension values of a key (NaN = not pushed) and its presence mask"""
    i01, i3, i4, i5, i6, i7, i8 = unpack(slots)
    fb, err, ended = i01 % 3, (i01 // 3) % 2, i01 // 6
    d = np.full(9, np.nan)
    d[0] = 1.0 if fb == 1 else (-1.0 if fb == 2 else 0.0)
    d[1] = 1.0 if fb == 1 else (-0.5 if err else (0.8 if ended else 0.5))
    mask = 3
    if i3 != 4:
        d[2] = np.array([d2bits], np.uint64).view(np.float64)[0]
        d[3], d[4] = LEVELS[3][i3], LEVELS[4][i4]
        mask |= 0x1C
    for g, i, bit in ((5, i5, 0x20), (6, i6, 0x40), (7, i7, 0x80), (8, i8, 0x100)):
        if i != ABSENT[g]:
            d[g] = LEVELS[g][i]
            mask |= bit
    return d, mask


def fx(v):
    """rint(v * 2^52) as an exact int (to_fx)"""
    return int(np.rint(np.float64(v) * 4503599627370496.0))


def weighted(dig, value_of):
    """sum count * value_of(d2 bits, slots) over the counted keys (value_of returns None for an uncounted key), exact ints"""
    s = n = 0
    for (d, k), c in dig.items():
        v = value_of(d, k)
        if v is not None:
            s += c * v
            n += c
    return s, n


def fixed_words(rep, idx_base):
    """the 45 fixed words of the digest from a report (the scan's words): tallies, byMode, pattern counts, tool totals,
    then per pattern its first three examples as inverted indices (0 = none)"""
    w = [rep.good, rep.bad, rep.none]
    for m in range(5):
        w += list(rep.byMode[m])
    w += [rep.pat[p].count if rep.bad else 0 for p in range(6)]
    w += [rep.toolCalls, rep.toolSucc, rep.toolFail]
    for p in range(6):
        for k in range(3):
            x = int(rep.pat[p].examples[k])
            w.append(0 if x < 0 else int(np.array([~np.uint64(x)], np.uint64).view(np.int64)[0]))
    return [int(x) for x in w]


def distinct_d2(T, seed):
    """T VALID records whose tool_success_rate values are almost all distinct (more than 2^20 distinct d2 keys at T = 2^22)"""
    from importlib import import_module
    dt = import_module("senweaver-ide_b200").RECORD_DTYPE
    rng = np.random.default_rng(seed)
    r = np.zeros(T, dt)
    r["toolCalls"] = rng.integers(1 << 20, 1 << 31, T, dtype=np.uint32)
    r["toolSucc"] = (r["toolCalls"].astype(np.uint64) * rng.integers(0, 1 << 20, T, dtype=np.uint64) >> np.uint64(20)).astype(np.uint32)
    r["feedback"] = rng.integers(0, 3, T)
    r["flags"] = 0x08 | rng.integers(0, 4, T)
    r["mode"] = rng.integers(0, 5, T)
    r["llmCalls"] = rng.integers(0, 9, T)
    r["tokens"] = rng.integers(0, 40000, T)
    r["userMsgs"] = rng.integers(0, 12, T)
    r["asstMsgs"] = rng.integers(0, 12, T)
    r["toolDurMs"] = rng.integers(0, 1 << 20, T).astype(np.float32)
    return r
