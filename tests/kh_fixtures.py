"""A plan model of K1h's launch (csrc/apo_tuple.cu run_reward9th / k_reward9th / kh_rows, csrc/apo_corpus.cuh cd_warp) and
Form D tensors whose Form T copy gets per-row dictionary counts that put that launch at its edges.

kh_plan restates the launch's arithmetic: the grid, each CTA's [lo, hi) of the pair array and [lo, hi) of the digest's
entries, the digest pass it takes (its last warp beside 992 streaming threads, or all 1024 threads and then the block-wide
pass), the ballot search for its first row round by round, and the row segments it streams.  Only the row lengths matter
to the launch, and a row's pair count is the number of distinct evaluations in it, so every tensor here is built from
rows of chosen lengths over one pool of distinct evaluations (test_gpu_twin_t_list.distinct):

- search: C in {1, 2, 32, 33, 1024, 1025, 4097} rows (0, 1, 1 - 2, 2, 3 and 3 search rounds), with the CTA cuts of forced
  grids of 2, 3, 7 and 13 CTAs and of the largest grid the pair count allows placed on a round's probe offset off[c] and
  one pair either side of it; the last row holding the last cut; one row under every CTA (C = 1, and C = 2 with a second
  row of one pair).  At C = 4097 the largest grid is the device's SM count.
- stride: rows of 7935, 7936, 7937 and 15 873 pairs (K1h streams 992 x 8 = 7936 pairs per round beside the digest warp)
  and 8191, 8192 and 8193 (1024 x 8 without it), whole inside one CTA at 2 CTAs, and at 7 CTAs rows that a CTA starts
  inside (s = lo) with those lengths left.
- digest: at 7 CTAs, CTAs of 128 * share - 1 and 128 * share pairs (first tensor) or 128 * share and 128 * share + 1
  (second), with digests of 7 s + 1 and 7 s + 6 entries (uneven shares: some CTAs take the block pass, others the warp's
  in one launch), 7 s (even shares) and 1 and 6 (fewer entries than CTAs: shares of 0).
- k3: rows of at most two distinct evaluations out of eight (a Form T copy with counts at any C), in tie groups, with
  rows of no counted evaluation (score -inf): C = k1_fixtures.k3_sizes(), whose finalising tail inside K1h ranks by
  counting up to C = 1024 (the digest's 8 KB LUT holds 1024 keys) and selects by radix from C = 1025 on.

Plain helpers, imported by the tests that use them (no fixtures, no GPU)."""
import bisect
import functools
from collections import namedtuple

import numpy as np

import flagship_fixtures as ff
import k1_fixtures as kf
import test_gpu_twin_t_list as tl

KH_THREADS = 1024                      # apo_tuple.cu
KH_UNROLL = 8
KH_PAIRS_PER_ENTRY = 128
NT_WARP = KH_THREADS - 32              # the streaming threads beside the digest warp
STRIDE_WARP, STRIDE_BLOCK = NT_WARP * KH_UNROLL, KH_THREADS * KH_UNROLL      # 7936, 8192 pairs per round of the stream
TAIL_SCRATCH_KEYS = 1024               # apo_corpus.cuh cd_tail: the LUT lent to the finaliser
H100_SMS = 132                         # the default grid of an H100 SXM; a device with fewer SMs only shortens it
GRIDS = (2, 3, 7, 13, None)            # APO_K1_GRID; None: the default (the device's SM count, capped by the pairs)

Cta = namedtuple("Cta", "k lo hi d_lo d_hi share block nt row rounds segs")
Plan = namedtuple("Plan", "grid nnz ctas")


# ------------------------------------------------------------------------------------------------ the plan model
def launched_grid(nnz, grid=None, sm=H100_SMS):
    """run_reward9th: the SM count, lowered by a forced grid, capped at one CTA per 1024 pairs, at least 1"""
    g = grid if grid and grid < sm else sm
    return max(1, min(g, -(-nnz // KH_THREADS)))


def search(off, C, lo):
    """kh_rows' ballot search for the row of pair lo: (row, [(a, b, step, winning lane)] per round).  The model asserts
    that it ends on the row bisect finds."""
    a, b, rounds = 0, C, []
    while b - a > 1:
        step = (b - a + 31) // 32
        le = 0
        for lane in range(32):
            i = a + lane * step
            if i < b and off[i] <= lo:
                le |= 1 << lane
        lane = le.bit_length() - 1                  # 31 - clz(le); lane 0 always votes
        rounds.append((a, b, step, lane))
        a += lane * step
        b = min(a + step, b)
    assert a == bisect.bisect_right(off, lo, 0, C + 1) - 1, (lo, a)
    return a, rounds


def kh_plan(nnz, off, cd_n, grid=None, corpus_on=True, sm=H100_SMS):
    """the launch of K1h over a pair array of nnz pairs in rows off [C + 1], with a digest of cd_n entries (0: a call
    without the corpus report, whose tail still rides on the launch), at a forced grid (None: the default).
    corpus_on=False: a session's accumulate or TUNE_NO_FUSE (no digest pass, no tail: 1024 streaming threads)."""
    off = [int(x) for x in off]
    C = len(off) - 1
    assert off[0] == 0 and off[C] == nnz
    g = launched_grid(nnz, grid, sm)
    ctas = []
    for k in range(g):
        lo, hi = nnz * k // g, nnz * (k + 1) // g
        d_lo, d_hi = cd_n * k // g, cd_n * (k + 1) // g
        share = d_hi - d_lo
        block = corpus_on and hi - lo < KH_PAIRS_PER_ENTRY * share
        nt = KH_THREADS if block or not corpus_on else NT_WARP
        row, rounds, segs = None, [], []
        if lo < hi:
            row, rounds = search(off, C, lo)
            for c in range(row, C):
                if off[c] >= hi:
                    break
                s, t = max(lo, off[c]), min(hi, off[c + 1])
                if s < t:
                    segs.append((c, s, t))
        ctas.append(Cta(k, lo, hi, d_lo, d_hi, share, block, nt, row, rounds, segs))
    return Plan(g, nnz, ctas)


def round_of(C, c):
    """the search round in which row c >= 1 is a probe point a + lane * step (lane >= 1) on the way to it"""
    a, b, r = 0, C, 0
    while b - a > 1:
        r += 1
        step = (b - a + 31) // 32
        lane = (c - a) // step
        a += lane * step
        b = min(a + step, b)
        if lane and a == c:
            return r
    return None


def search_rounds(C):
    return max([round_of(C, c) or 0 for c in range(C)] or [0])


def probe_hits(plan, off):
    """{(round, d)}: interior cuts lo that lie at d in {-1, 0, +1} from the offset of a probe point (lane >= 1) of a round
    of their own search"""
    hits = set()
    for cta in plan.ctas[1:]:
        for r, (a, b, step, _) in enumerate(cta.rounds, 1):
            for lane in range(1, 32):
                i = a + lane * step
                if i < b and cta.lo - int(off[i]) in (-1, 0, 1):
                    hits.add((r, cta.lo - int(off[i])))
    return hits


# ------------------------------------------------------------------------------------------------ rows of chosen lengths
POOL_N = 16_500


@functools.lru_cache(maxsize=1)
def pool():
    return tl.distinct(0x5EEDF200, POOL_N, tl.zero_weight_rows())


def lengths_of(off):
    return np.diff(np.asarray(off, np.int64))


def gate_T(off):
    """the fewest evaluations per row that hold every row's distinct evaluations and keep the counts (8 nnz <= C T / 2)"""
    ln = lengths_of(off)
    C, nnz = len(ln), int(ln.sum())
    return max(int(ln.max()), -(-16 * nnz // C))


def rows_dims(off, seed, T=None):
    """[C][T] dims whose row c holds exactly off[c + 1] - off[c] distinct evaluations of the pool (each at least once, the
    rest of the row repeats them)"""
    ln = lengths_of(off)
    T = gate_T(off) if T is None else T
    assert T >= ln.max() and ln.max() <= POOL_N
    rng = np.random.default_rng(seed)
    idx = np.empty((len(ln), T), np.int32)
    for c, L in enumerate(ln):
        ent = (c * 7919 + np.arange(L)) % POOL_N
        row = np.concatenate([ent, ent[rng.integers(0, L, T - L)]])
        idx[c] = row[rng.permutation(T)]
    return pool()[idx]


Fixture = namedtuple("Fixture", "name off K")


def fixture_dims(fx, seed=0x5EEDF201):
    return rows_dims(fx.off, seed + len(fx.off))


def _fill(C, nnz, pins):
    """off [C + 1] through the pins {c: off[c]}, the rows between two pins as even as they allow"""
    pts = sorted({0: 0, C: nnz, **pins}.items())
    off = np.empty(C + 1, np.int64)
    for (c0, v0), (c1, v1) in zip(pts, pts[1:]):
        off[c0:c1 + 1] = v0 + (v1 - v0) * np.arange(c1 - c0 + 1) // (c1 - c0)
    return off


def _fits(C, nnz, pins, c, v):
    """off[c] = v keeps at least two pairs per row between it and its neighbouring pins"""
    if not 0 < c < C or c in pins:
        return False
    pts = {0: 0, C: nnz, **pins}
    below = max(x for x in pts if x < c)
    above = min(x for x in pts if x > c)
    return v - pts[below] >= 2 * (c - below) and pts[above] - v >= 2 * (above - c)


def search_offsets(C, nnz, last_row=False, sm=H100_SMS):
    """row offsets whose CTA cuts at every grid of GRIDS land, in turn, on a probe offset of each search round and one pair
    either side (where the rows allow); last_row: the last row holds the last cut of the largest grid"""
    pins = {}
    if last_row:
        G = launched_grid(nnz, None, sm)
        pins[C - 1] = nnz - (nnz // G + nnz // (4 * G) + 2)
    R = search_rounds(C)
    kinds = [(r, d) for r in range(1, R + 1) for d in (0, -1, 1)]
    i = 0
    for grid in GRIDS:
        g = launched_grid(nnz, grid, sm)
        for k in range(1, g):
            if not kinds:
                break
            lo = nnz * k // g
            off = _fill(C, nnz, pins)
            nat = bisect.bisect_right(list(off), lo) - 1
            for j in range(len(kinds)):
                r, d = kinds[(i + j) % len(kinds)]
                c = next((c for dc in range(300) for c in (nat + dc, nat - dc)
                          if 0 < c < C and round_of(C, c) == r and _fits(C, nnz, pins, c, lo - d)), None)
                if c is not None:
                    pins[c] = lo - d
                    break
            i += 1
    return _fill(C, nnz, pins)


# (C, pairs, the last row holds the last cut): nnz > 13 * 1024 so that a forced grid of 13 is launched; at C = 4097 about
# 40 pairs per row give more than 132 * 1024 pairs (the default grid is the SM count)
SEARCH = (("c1", 1, 14_000, False), ("c32", 32, 16_000, True), ("c33", 33, 16_000, True), ("c1024", 1024, 20_000, True),
          ("c1025", 1025, 20_000, True), ("c4097", 4097, 4097 * 40, False))


@functools.lru_cache(maxsize=None)
def search_fixtures():
    out = [Fixture(name, search_offsets(C, nnz, last) if C > 1 else np.array([0, nnz], np.int64), min(4, C))
           for name, C, nnz, last in SEARCH]
    nnz = 14_000
    out.insert(1, Fixture("c2_half", np.array([0, nnz // 2, nnz], np.int64), 2))          # the cut of 2 CTAs on off[1]
    out.insert(2, Fixture("c2_spans", np.array([0, nnz - 1, nnz], np.int64), 2))           # row 0 under every CTA
    return out


# ------------------------------------------------------------------------------------------------ stride edges
STRIDE_ROWS = (7935, 7936, 7937, 15873, 8191, 8192, 8193)
STRIDE_MID = (7935, 7936, 7937, 15873, 8192, 8193)        # what is left of a row a CTA of 7 starts inside
MID_GRID, MID_BEFORE = 7, 40


def _off(lengths):
    return np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)


def _fillers(n, size=500):
    k = -(-n // size)
    return [n * (i + 1) // k - n * i // k for i in range(k)]


def stride_whole():
    """the stride rows, the cut of 2 CTAs inside a filler row between them: every stride row whole inside one CTA"""
    return _off([300, 15873, 8193, 8192, 600, 7935, 7936, 7937, 8191, 300])


def stride_mid():
    """at 7 CTAs of 16 500 pairs, cut k inside a row that starts MID_BEFORE pairs before it and has STRIDE_MID[k - 1]
    pairs left after it; filler rows of <= 500 pairs between"""
    nnz = 7 * 16_500
    lengths, pos = [], 0
    for k, L in enumerate(STRIDE_MID, 1):
        lo = nnz * k // MID_GRID
        lengths += _fillers(lo - MID_BEFORE - pos)
        lengths.append(MID_BEFORE + L)
        pos = lo + L
    lengths += _fillers(nnz - pos)
    return _off(lengths)


@functools.lru_cache(maxsize=None)
def stride_fixtures():
    return [Fixture("stride_whole", stride_whole(), 3), Fixture("stride_mid", stride_mid(), 3)]


# ------------------------------------------------------------------------------------------------ digest shares
DIG_GRID, DIG_S, DIG_ROWS = 7, 20, 16
DIG_KEYS = (1, 6, 7 * DIG_S, 7 * DIG_S + 1, 7 * DIG_S + 6)     # entries of the digests at DIG_GRID
IDX_BASE = 11


def digest_offsets(delta):
    """7 CTAs of 128 s + delta pairs, three of them (CTAs 2, 4, 6) one more"""
    nnz = DIG_GRID * (KH_PAIRS_PER_ENTRY * DIG_S + delta) + 3
    return _fill(DIG_ROWS, nnz, {})


@functools.lru_cache(maxsize=None)
def digest_fixtures():
    return [Fixture("digest_m1", digest_offsets(-1), 3), Fixture("digest_0", digest_offsets(0), 3)]


def digest_corpus(nkeys):
    return ff.cycled(ff.FEW_T, nkeys)


ROW_KEYS = 97                          # the digest beside the search and stride tensors


# ------------------------------------------------------------------------------------------------ K3 through K1h
K3_T, K3_POOL = 32, 8
K3_MODES = ("mixed", "sparse", "equal")
K3_ALL_MODES = (1025, 2049, 4096)


@functools.lru_cache(maxsize=1)
def k3_pool():
    p = tl.distinct(0x5EEDF202, K3_POOL, tl.zero_weight_rows())
    assert not np.isnan(p).all(axis=1).any()
    return np.concatenate([p, np.full((1, 9), np.nan, np.float32)])        # index K3_POOL: counted by no weight


def k3_index(C, mode="mixed"):
    """[C][K3_T] pool indices: equal, every row the same; mixed, by c mod 17: 16 no counted evaluation, 0 .. 5 one tie
    group each, the rest a copies of one evaluation and K3_T - a of another (distinct scores, and ties among repeats);
    sparse, 3 of 4 rows as mixed class 16"""
    idx = np.empty((C, K3_T), np.int64)
    for c in range(C):
        cls = 0 if mode == "equal" else 16 if mode == "sparse" and c % 4 else c % 17
        if cls == 16:
            x, y, a = K3_POOL, K3_POOL, K3_T
        elif cls < 6:
            x, y, a = cls, cls + 2, K3_T // 2
        else:
            x, y, a = c % K3_POOL, (c + 3) % K3_POOL, 1 + (c * 7) % K3_T
        idx[c] = np.where(np.arange(K3_T) < a, x, y)
    return idx


def k3_dims(C, mode="mixed"):
    return k3_pool()[k3_index(C, mode)]


def k3_cases():
    return [(C, m) for C in kf.k3_sizes() for m in (K3_MODES if C in K3_ALL_MODES else ("mixed",))]


def k3_offsets(C, mode="mixed"):
    """the row offsets of the copy's counts: one pair per distinct pool index of a row"""
    return _off([len(np.unique(r)) for r in k3_index(C, mode)])


def tail_select(C):
    """the top-K of K1h's finalising CTA: a counting rank over the keys in the lent LUT, or the radix select"""
    return "rank" if C <= TAIL_SCRATCH_KEYS else "radix"
