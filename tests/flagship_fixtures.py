"""Hand-built inputs that reach the edges of the flagship step's one launch: K1h (csrc/apo_tuple.cu k_reward9th) over the
per-row dictionary counts of the Form T copy (csrc/apo_abi.cu build_twin_h, k_th_count / k_th_rows), and the corpus digest
K1h and k_corpus_digest read (build_digest_buffers, csrc/apo_kernels.cu k_cd_count / cd_insert / k_cd_compact).

Form D tensors, all made of distinct evaluations Form T can index (test_gpu_twin_t_list.distinct):
- cap: a dictionary of exactly 2^20 entries (the copy's cap, and the 20-bit entry field of a pair) over C = 150 rows of
  T = 2^17 + 3: the count build's scratch takes R = 64 rows, so three batches, the last ragged (22 rows); one evaluation
  occurs once and is the rarest, so it is entry 2^20 - 1.  over_cap: one more distinct evaluation, no copy.
- two_batches: C = 128 rows over a dictionary that again gives R = 64: two full batches.
- chunks: evaluation counts chosen so that entries 31 / 32 (a thread's 32-entry slice of k_th_rows), 8191 / 8192 and
  16383 / 16384 (its 8192-entry chunks) are single, known evaluations, whatever the dictionary's order among equal counts;
  one row holds a single pair in the last chunk.
- nnz_gate: 8 nnz == C T / 2 (counts held) and one pair more (none held).
- wide: rows of 2^25 evaluations of +-(2 - 2^-23) in one dimension (table values about +-2^53): per-row sums past 2^64
  that cancel to a small remainder, and a row of a single entry.

Corpora for the digest (apo_record arrays), whose distinct VALID reward keys (corpus_digest_model) are counted by design:
each key k is a record template (mode, feedback, flags by k mod 5) with toolSucc = k out of toolCalls = 2^24, so its d2
is exact and distinct per k:
- gate_small / gate_large: exactly the digest's cap of keys (kept) and one more (dropped), at T = 2^20 (cap 2^18) and
  T = 2^22 + 5 (cap 2^20); and the cap's keys plus many more on records without VALID (kept).
- no_valid: 2^20 + 3 records, none VALID: a digest of no entries.
- probe: keys whose home slot in cd_insert's table is one slot (a chain of ~256) or the last slot (their probes wrap to
  slot 0), found once by find_probe_keys() and kept in tests/golden/digest_probe_keys.json.
- few: 1, 2 and 7 keys, fewer entries than K1h has CTAs.

Plain helpers, imported by the tests that use them (no fixtures, no GPU)."""
import json
import os

import numpy as np

import oracle
import test_gpu_twin_t_list as tl

HERE = os.path.dirname(os.path.abspath(__file__))

# ------------------------------------------------------------------------------------------------ the count build
COUNT_SHIFT = 20                       # apo_kernels.h KH_COUNT_SHIFT
TWIN_T_CAP = 1 << 20                   # apo_abi.cu kTwinTCap
H_SCRATCH = 256 << 20                  # apo_abi.cu kTwinHScratch
TH_CHUNK = 8192                        # apo_tuple.cu TH_CHUNK
KT_HOT_MAX = 24576                     # apo_kernels.h


def batches(n, C):
    """build_twin_h's batching for a dictionary of n entries over C rows: (npitch, rows per batch R, batches, last batch)"""
    npitch = -(-n // 32) * 32
    R = min(C, max(1, H_SCRATCH // (4 * npitch)))
    nb = -(-C // R)
    return npitch, R, nb, C - (nb - 1) * R


def counts_held(nnz, C, T):
    """build_twin_h's gate: the counts take at most a quarter of K1t2's slot plane"""
    return 8 * nnz <= C * T // 2


def rank_index(idx):
    """[C][T] pool indices -> (dictionary index per evaluation, count per pool entry) in the copy's order: count descending;
    equal counts in pool order (the engine orders them by tuple key: only entries of a count no other entry has get the
    same index from both)"""
    n = int(idx.max()) + 1
    cnt = np.bincount(idx.reshape(-1), minlength=n)
    order = np.lexsort((np.arange(n), -cnt))
    rank = np.empty(n, np.int64)
    rank[order] = np.arange(n)
    return rank[idx], cnt


def fixed_rank(cnt, i):
    """the dictionary index entry i gets in any order that ranks by count descending, when its count is unique (else None)"""
    if np.count_nonzero(cnt == cnt[i]) != 1:
        return None
    return int(np.count_nonzero(cnt > cnt[i]))


def _dict_rows(seed, C, T, head, tails, single_row):
    """[C][T] pool indices: every row draws from a shared head of `head` entries, and row c holds its own tail entries
    tails[c] (disjoint ranges of the pool after the head) twice each, except the first tail entry of single_row, held once"""
    rng = np.random.default_rng(seed)
    idx = np.empty((C, T), np.int64)
    for c in range(C):
        t = tails[c]
        reps = np.full(len(t), 2)
        if c == single_row:
            reps[0] = 1
        own = np.repeat(t, reps)
        assert len(own) + head <= T
        row = np.concatenate([np.arange(head), own, rng.integers(0, head, T - head - len(own))])
        idx[c] = row[rng.permutation(T)]
    return idx


def _pool(seed, n):
    return tl.distinct(seed, n, tl.zero_weight_rows())


CAP_C, CAP_T, CAP_HEAD, CAP_SINGLE_ROW = 150, (1 << 17) + 3, 256, 149


def _cap_tails():
    return np.array_split(np.arange(CAP_HEAD, TWIN_T_CAP), CAP_C)


CAP_SINGLE = int(_cap_tails()[CAP_SINGLE_ROW][0])          # the pool entry seen once: entry 2^20 - 1, in the ragged batch


def cap_index():
    """[150][2^17 + 3] pool indices over exactly 2^20 distinct entries; pool entry CAP_SINGLE is the one seen once"""
    return _dict_rows(0x5EEDF100, CAP_C, CAP_T, CAP_HEAD, _cap_tails(), CAP_SINGLE_ROW)


def over_cap_index(idx):
    """the cap indices with one head evaluation of the last row replaced by pool entry 2^20, a new distinct evaluation"""
    i = idx.copy()
    i[-1, int(np.flatnonzero(idx[-1] < CAP_HEAD)[0])] = TWIN_T_CAP
    return i


def cap(over=False):
    """(dims, pool indices): the dictionary at the copy's cap, or (over) one entry past it"""
    idx = cap_index()
    if over:
        idx = over_cap_index(idx)
    return _pool(0x5EEDF100, TWIN_T_CAP + 1)[idx], idx


TWO_C, TWO_HEAD, TWO_TAIL = 128, 32, 8150


def two_batches():
    """(dims, pool indices): 128 rows of 2^17 + 3 over 32 + 128 * 8150 entries (R = 64: two full batches)"""
    tails = [TWO_HEAD + np.arange(c * TWO_TAIL, (c + 1) * TWO_TAIL) for c in range(TWO_C)]
    idx = _dict_rows(0x5EEDF101, TWO_C, CAP_T, TWO_HEAD, tails, None)
    pool = _pool(0x5EEDF101, TWO_HEAD + TWO_C * TWO_TAIL)
    return pool[idx], idx


# chunks: 31 filler entries (the most frequent: indices 0..30), then entries of unique counts at the edges and two groups of
# equal counts between them; every evaluation of an edge entry or a group entry lies in one row
CH_C, CH_T = 8, 40_003
CH_EDGES = {31: 8, 32: 7, 8191: 5, 8192: 4, 16383: 2, 16384: 1}      # dictionary index -> its count
CH_GROUPS = ((33, 8191, 6), (8193, 16383, 3))                          # [first, end) indices, count of each


def chunks():
    """(dims, pool indices, {dictionary index: pool entry} of the edge entries).  Row 0: the filler and entry 16384 alone in
    the last chunk; row 1: the filler and entries 31, 32, 8191, 8192, 16383; rows 2..7: the two groups, dealt out whole"""
    rng = np.random.default_rng(0x5EEDF102)
    n = 16385
    pool_of = {}                                  # pool entry p: filler 0..30, edges next, then the groups
    p = 31
    for e in CH_EDGES:
        pool_of[e] = p
        p += 1
    group = []
    for first, end, k in CH_GROUPS:
        group.append((np.arange(p, p + end - first), k))
        p += end - first
    assert p == n
    rows = [[np.array([pool_of[16384]])],
            [np.repeat(pool_of[e], CH_EDGES[e]) for e in (31, 32, 8191, 8192, 16383)]]
    for c in range(CH_C - 2):                     # whole entries per row: an entry's evaluations stay in one row
        rows.append([np.repeat(np.array_split(ent, CH_C - 2)[c], k) for ent, k in group])
    idx = np.empty((CH_C, CH_T), np.int64)
    for c, parts in enumerate(rows):
        own = np.concatenate(parts)
        fill = np.concatenate([np.arange(31), rng.integers(0, 31, CH_T - len(own) - 31)])
        r = np.concatenate([own, fill])
        idx[c] = r[rng.permutation(CH_T)]
    pool = _pool(0x5EEDF102, n)
    return pool[idx], idx, pool_of


NNZ_C, NNZ_T = 4, 16_004                          # C T / 16 = 4001 pairs: 1000, 1000, 1000, 1001


def nnz_gate(extra):
    """(dims, pool indices) with 8 nnz == C T / 2 (extra = 0: counts held) or one pair more (extra = 1: none held)"""
    rng = np.random.default_rng(0x5EEDF103)
    per = (1000, 1000, 1000, 1001)
    pool = _pool(0x5EEDF103, 1400)
    idx = np.empty((NNZ_C, NNZ_T), np.int64)
    for c, k in enumerate(per):
        ent = np.arange(100 * c, 100 * c + k)
        r = np.concatenate([ent, rng.choice(ent, NNZ_T - k)])
        idx[c] = r[rng.permutation(NNZ_T)]
    if extra:
        t = int(np.flatnonzero(idx[0] == idx[0, -1])[0])      # an entry row 0 holds more than once
        idx[0, t] = 1399
    return pool[idx], idx


WIDE_T = 1 << 25
WIDE_MAX = np.float32(np.nextafter(np.float32(2), np.float32(0)))        # 2 - 2^-23
WIDE_SPLIT = ((1 << 24) + 3, (1 << 24) - 3)                               # row 0: +, - evaluations


def wide_rows():
    """the two distinct evaluations of wide(): [2][9] (+, -)"""
    d = np.full((2, 9), np.nan, np.float32)
    d[0, 0], d[1, 0] = WIDE_MAX, -WIDE_MAX
    return d


def wide():
    """[2][2^25][9]: row 0 holds 2^24 + 3 evaluations of +(2 - 2^-23) and 2^24 - 3 of -(2 - 2^-23), interleaved in runs;
    row 1 holds only the + one"""
    e = wide_rows()
    d = np.empty((2, WIDE_T, 9), np.float32)
    sign = (np.arange(WIDE_T) // 4) % 2 == 1                                # True: the - evaluation, in runs of 4 ...
    sign[-8:] = [False, True] + [False] * 6                                 # ... then 7 + and one -
    assert WIDE_T - sign.sum() == WIDE_SPLIT[0]
    d[0] = e[0]
    d[0, sign] = e[1]
    d[1] = e[0]
    return d


def wide_counts():
    """per row, the count of each of the two distinct evaluations"""
    return [WIDE_SPLIT, (WIDE_T, 0)]


# ------------------------------------------------------------------------------------------------ the digest
F_ERRORS, F_ENDED, F_VALID = 0x01, 0x02, 0x08
KEY_CALLS = 1 << 24
DIGEST_MIN, DIGEST_CAP, DIGEST_SPILL = 1 << 20, 1 << 20, 1 << 20        # apo_abi.cu kDigestMinRecords / Cap / Spill
GOLD = 0x9E3779B97F4A7C15
M64 = (1 << 64) - 1


def digest_cap(T):
    return min(DIGEST_CAP, T // 4)


def digest_slots(T):
    """build_digest_buffers' table size"""
    s = 1024
    while s < 2 * digest_cap(T) + DIGEST_SPILL:
        s <<= 1
    return s


def mix64(z):
    """apo_device.cuh mix64 on Python ints"""
    z &= M64
    z ^= z >> 30
    z = (z * 0xBF58476D1CE4E5B9) & M64
    z ^= z >> 27
    z = (z * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def home_slot(d2bits, slots, nslots):
    """cd_insert's first probe for the key {d2 bits, slots}"""
    return mix64(int(d2bits) ^ mix64(int(slots) + GOLD)) & (nslots - 1)


def keyed(k, valid=None, calls=KEY_CALLS, template=None):
    """one record per element of k (key numbers): template k mod 5 unless given (mode, feedback, flags, counters), toolSucc
    = k out of toolCalls = calls; valid: bool per record (default all VALID)"""
    k = np.asarray(k, np.int64)
    r = np.zeros(len(k), oracle.RECORD_DTYPE)
    j = k % 5 if template is None else np.full(len(k), template)
    r["mode"] = j
    r["feedback"] = np.array([0, 1, 2, 2, 1])[j]
    r["flags"] = F_ENDED | np.array([0, 0, F_ERRORS, 0, F_ERRORS])[j]
    r["userMsgs"] = np.array([1, 3, 8, 2, 12])[j]
    r["asstMsgs"] = np.array([1, 4, 9, 2, 12])[j]
    r["llmCalls"] = np.array([1, 2, 5, 3, 9])[j]
    r["tokens"] = np.array([500, 3000, 12_000, 40_000, 800])[j]
    r["toolDurMs"] = np.array([100.0, 0.0, 5000.0, 2.0e10, 1.0], np.float32)[j]
    r["toolCalls"] = calls
    r["toolSucc"] = k
    r["toolFail"] = np.array([0, 1, 3, 6, 0])[j]
    valid = np.ones(len(k), bool) if valid is None else np.asarray(valid, bool)
    r["flags"] |= np.where(valid, F_VALID, 0).astype(np.uint8)
    return r


def cycled(T, nkeys):
    """T records cycling through keys 0 .. nkeys - 1"""
    return keyed(np.arange(T) % nkeys)


GATE_SMALL_T = 1 << 20                  # cap 2^18
GATE_LARGE_T = (1 << 22) + 5            # cap 2^20


def gate(T, extra):
    """exactly digest_cap(T) distinct VALID keys (kept), or one more (extra = 1: dropped)"""
    return cycled(T, digest_cap(T) + extra)


def gate_invalid(T):
    """digest_cap(T) VALID keys on the even records; on the odd ones a distinct key each, without VALID (kept)"""
    t = np.arange(T)
    k = np.where(t % 2 == 0, (t // 2) % digest_cap(T), digest_cap(T) + t // 2)
    return keyed(k, valid=t % 2 == 0)


NO_VALID_T = (1 << 20) + 3


def no_valid():
    return keyed(np.arange(NO_VALID_T) % 1000, valid=np.zeros(NO_VALID_T, bool))


PROBE_T = (1 << 20) + 7                 # cap 2^18 + 1, a table of 2^21 slots
PROBE_CALLS = 1 << 31                   # the probe keys: toolSucc k out of 2^31 calls, template 0
PROBE_GOLDEN = os.path.join(HERE, "golden", "digest_probe_keys.json")


def probe_golden():
    with open(PROBE_GOLDEN) as f:
        return json.load(f)


def probe():
    """(records, chain keys, wrap keys): each probe key (toolSucc out of PROBE_CALLS) on 3 records, then filler records
    cycling through 5000 keys of the usual form"""
    g = probe_golden()
    chain, wrap = g["chain"], g["wrap"]
    pk = np.array(chain + wrap, np.int64)
    filler = cycled(PROBE_T - 3 * len(pk), 5000)
    recs = np.concatenate([np.repeat(keyed(pk, calls=PROBE_CALLS, template=0), 3), filler])
    return recs[np.random.default_rng(0x5EEDF104).permutation(len(recs))], chain, wrap


def probe_slots():
    """the slots half of every probe key"""
    import corpus_digest_model as dm
    return int(dm.keys(keyed([0], calls=PROBE_CALLS, template=0))[1][0])


def find_probe_keys(target, nslots, n_chain=256, n_wrap=64, step=1 << 25):
    """toolSucc values k < 2^31 whose probe key's home slot is `target` (n_chain of them) or nslots - 1 (n_wrap): a numpy
    search of about twenty seconds, whose result PROBE_GOLDEN keeps"""
    hy = np.uint64(mix64(probe_slots() + GOLD))
    mask = np.uint64(nslots - 1)
    chain, wrap = [], []

    def mix(z):
        z = z ^ (z >> np.uint64(30)); z = z * np.uint64(0xBF58476D1CE4E5B9)
        z = z ^ (z >> np.uint64(27)); z = z * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))
    with np.errstate(over="ignore"):
        for a in range(0, PROBE_CALLS, step):
            k = np.arange(a, a + step, dtype=np.int64)
            x = ((k.astype(np.float64) / float(PROBE_CALLS)) * 2.0 - 1.0).view(np.uint64)
            h = mix(x ^ hy) & mask
            chain += k[h == np.uint64(target)].tolist()
            wrap += k[h == mask].tolist()
            if len(chain) >= n_chain and len(wrap) >= n_wrap:
                break
    return chain[:n_chain], wrap[:n_wrap]


FEW = (1, 2, 7)
FEW_T = (1 << 20) + 9


def few(nkeys):
    return cycled(FEW_T, nkeys)
