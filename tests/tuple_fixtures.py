"""Hand-built Form T tensors that reach the edges of k_tuple_values and K1t (csrc/apo_tuple.cu), and the one plain reference
they are checked against.

Unlike the encoder's output (apo_tuple_encode_host: most frequent entry first, tens of thousands of entries at test sizes),
the dictionaries here have chosen sizes -- around the shared-memory head (hot = min(n + 1, 24576)), where the high index
plane th becomes non-zero (65536), 2^20 + 3 and APO_TUPLES_MAX = 2^24 - 1 -- and the index planes put chosen indices at
chosen positions:

- codebook() / d2book(): the two Form P codebooks.  Codes 0..10 of every coded dimension hold ordinary values in [-1, 1];
  codes 11..14 hold the special values of SPECIAL_SLOTS (+-(2 - 2^-23), +-2.0, a NaN value) or stay empty (0xFFFFFFFF, as
  apo_packed_encode_host leaves unused slots).  d2book slots 0..4092 hold distinct values, 4093 is empty, 4094 a NaN value.
- dictionary(n): n DISTINCT Form P pairs.  Entry i is built from i mod 4093 (its tool_success_rate index; 4093 is prime) and
  i div 4093 (base-12 digits of a multiple of it as the eight codes), so flipping or dropping any index bit changes the
  tool_success_rate index and therefore the value: no entry value repeats with a power-of-two period in the index.  The
  entries of ENTRIES (maximal values, nulls, refused entries) can be placed at chosen indices.
- the index-plane builders (PLANES): every 8-evaluation group with 8 different high bytes, boundary indices at fixed
  positions, whole warps on one entry, uniform, reversed frequency, one shared-memory bank pair; and groups of maximal
  entries (max_groups).
- entry_fx() / expected(): the reference.  Entries are decoded through the codebooks into Form D fp32 rows (absent = NaN),
  scored one evaluation per "candidate" by oracle.score_dims_fx (IEEE division in C), and the per-candidate sums are exact
  integers (two int64 halves of fx, recombined as Python ints).

Plain helpers, imported by the tests that use them (no fixtures, no GPU)."""
import ctypes as C

import numpy as np

import oracle

TILE = 8192                         # K1t tile (KT_TILE): rows end in a ragged tile read by the scalar loop
HOT_MAX = 24576                     # KT_HOT_MAX: dictionary entries served from shared memory
TUPLES_MAX = 0xFFFFFF               # APO_TUPLES_MAX
SIZES = (1, 2, 24574, 24575, 24576, 24577, 65535, 65536, 65537, (1 << 20) + 3, TUPLES_MAX)
T_EDGES = (1, 7, 8, 8191, 8192, 8193, 16385)
P_D2 = 4093                         # prime: tool_success_rate index of bulk entry i is i mod P_D2
NB = 11                             # bulk codes per coded dimension (0..10); base-12 digit 11 = absent
MIX = 7919                          # i div P_D2 is multiplied by this before its base-12 digits become the codes
EMPTY = 0xFFFFFFFF                  # an unused codebook slot
NAN_VALUE = 0x7FC00001              # a NaN value that is not the empty pattern
MAXV = np.float32(2 - 2 ** -23)     # largest fp32 below 2
D2_EMPTY, D2_NAN, D2_ABSENT = 4093, 4094, 4095
ABSENT = 15

# (coded dimension j, code) -> fp32 value of the special slots; every other slot >= NB is empty
SPECIAL_SLOTS = {(7, 11): MAXV, (7, 12): -MAXV, (7, 13): np.float32(2.0), (7, 14): np.float32(-2.0),
                 (6, 11): MAXV, (6, 12): -MAXV}
CODE_NAN, CODE_EMPTY = (5, 11), (5, 12)

# dimensions 0 and 3 have weight 0 here: an entry with only those present is null (total weight 0)
ZERO_W = np.array([0.0, 0.4, 0.05, 0.0, 0.1, 0.1, 0.15, 0.1, 0.1])
# total weight with an all-ones significand: k_tuple_values takes the IEEE division (__ddiv_rn)
ONES_W = np.array([0.3, 0.1, 0.05, 0.05, 0.1, 0.1, 0.1, 0.1, 0.1])


def _bits(f) -> int:
    return int(np.float32(f).view(np.uint32))


def codebook() -> np.ndarray:
    """[8 * 256] uint32: codes 0..10 ordinary distinct values per dimension, then SPECIAL_SLOTS, the NaN value, empties"""
    book = np.full((8, 256), EMPTY, np.uint32)
    for j in range(8):
        vals = ((np.arange(NB) * 7 + 3 * j) % NB - 5) / 5.0 * (1 - j / 64)
        book[j, :NB] = vals.astype(np.float32).view(np.uint32)
    for (j, c), v in SPECIAL_SLOTS.items():
        book[j, c] = _bits(v)
    book[CODE_NAN] = NAN_VALUE
    return book.reshape(-1)


def d2book() -> np.ndarray:
    book = np.full(4096, EMPTY, np.uint32)
    book[:P_D2] = (-1.0 + 2.0 * np.arange(P_D2) / (P_D2 - 1)).astype(np.float32).view(np.uint32)
    book[D2_NAN] = NAN_VALUE + 1
    return book


def pack_pc(codes) -> int:
    """{coded dimension j: code} -> Form P code word (absent dimensions 15)"""
    w = 0
    for j in range(8):
        w |= codes.get(j, ABSENT) << (4 * j)
    return w


# named entries (pc, pd): GOOD ones are scored, BAD ones must fail the call with APO_E_ARG
ENTRIES = {
    "pmax": (pack_pc({7: 11}), D2_ABSENT),          # finalReward = +(2 - 2^-23): one present dimension
    "nmax": (pack_pc({7: 12}), D2_ABSENT),
    "pmax6": (pack_pc({6: 11}), D2_ABSENT),
    "nmax6": (pack_pc({6: 12}), D2_ABSENT),
    "null": (0xFFFFFFFF, D2_ABSENT),                # mask 0
    "zw": (pack_pc({0: 0, 2: 0}), D2_ABSENT),       # dimensions 0 and 3 only: null under ZERO_W
    "p2": (pack_pc({7: 13}), D2_ABSENT),            # finalReward = +2.0 exactly
    "n2": (pack_pc({7: 14}), D2_ABSENT),
    "d2_empty": (pack_pc({j: 0 for j in range(8)}), D2_EMPTY),
    "d2_nan": (pack_pc({j: 0 for j in range(8)}), D2_NAN),
    "code_empty": (pack_pc({CODE_EMPTY[0]: CODE_EMPTY[1]}), 0),
    "code_nan": (pack_pc({CODE_NAN[0]: CODE_NAN[1]}), 0),
}
GOOD = ("pmax", "nmax", "pmax6", "nmax6", "null", "zw")
BAD = ("p2", "n2", "d2_empty", "d2_nan", "code_empty", "code_nan")


def hot(n: int) -> int:
    return min(n + 1, HOT_MAX)


def default_places(n: int) -> dict:
    """where the GOOD entries sit: the maximal ones in the head (1, 2) and at the end of the dictionary (the tail once n > hot),
    the nulls at 3 and n - 5; nothing below 16 entries"""
    if n < 16:
        return {}
    return {"pmax": 1, "nmax": 2, "null": 3, "pmax6": n - 3, "nmax6": n - 2, "zw": n - 5}


def bulk(i: np.ndarray):
    """(pc, pd) of bulk entry i: pd = i mod P_D2, codes = base-12 digits of (i div P_D2) * MIX (digit 11 -> absent)"""
    i = np.asarray(i, np.int64)
    pd = (i % P_D2).astype(np.uint16)
    b = (i // P_D2) * MIX
    pc = np.zeros(i.shape, np.uint32)
    for j in range(8):
        d = (b // 12 ** j) % 12
        pc |= (np.where(d < NB, d, ABSENT).astype(np.uint32) << np.uint32(4 * j))
    return pc, pd


def dictionary(n: int, places=None):
    """n distinct Form P pairs (tb_pc uint32[n], tb_pd uint16[n]); places = {entry name: index} (default_places(n) if None)"""
    pc, pd = bulk(np.arange(n))
    for name, i in (default_places(n) if places is None else places).items():
        pc[i], pd[i] = ENTRIES[name]
    return pc, pd


def decode(tbook, book, d2b) -> np.ndarray:
    """dictionary entries -> Form D fp32 rows [n][9] (absent and empty / NaN slots as NaN), vectorised"""
    pc, pd = tbook
    vals = book.reshape(8, 256).view(np.float32)
    out = np.full((len(pc), 9), np.nan, np.float32)
    for j, dim in enumerate((0, 1, 3, 4, 5, 6, 7, 8)):
        code = (pc >> np.uint32(4 * j)) & np.uint32(15)
        present = code != ABSENT
        out[present, dim] = vals[j][code[present]]
    k2 = pd & np.uint16(4095)
    p2 = k2 != D2_ABSENT
    out[p2, 2] = d2b.view(np.float32)[k2[p2]]
    return out


def entry_fx(tbook, book, d2b, w=None, chunk=1 << 20):
    """(fx int64[n], counted uint8[n]) of every entry: oracle.score_dims_fx on shape [n, 1, 9], in chunks"""
    L = oracle.lib()
    w = oracle.weights() if w is None else np.ascontiguousarray(w, np.float64)
    n = len(tbook[0])
    fx, counted = np.empty(n, np.int64), np.empty(n, np.uint8)
    for a in range(0, n, chunk):
        b = min(n, a + chunk)
        rows = np.ascontiguousarray(decode((tbook[0][a:b], tbook[1][a:b]), book, d2b).reshape(b - a, 1, 9))
        lo, hi, cnt = np.empty(b - a, np.uint64), np.empty(b - a, np.int64), np.empty(b - a, np.uint64)
        L.orc_score_dims_fx(rows.ctypes.data_as(C.c_void_p), b - a, 1, 1, w.ctypes.data_as(C.c_void_p),
                            lo.ctypes.data_as(C.c_void_p), hi.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p))
        v = lo.view(np.int64)
        assert np.array_equal(hi, v >> 63)                  # one evaluation: the 128-bit sum is its sign-extended fx
        fx[a:b], counted[a:b] = v, cnt
    return fx, counted


def expected(idx: np.ndarray, fx: np.ndarray, counted: np.ndarray):
    """exact per-candidate (sums, counts) of index rows idx [C][T] (indices < n): int64 halves of fx summed, recombined"""
    sums, counts = [], []
    for row in np.asarray(idx).reshape(len(idx), -1):
        v = fx[row]
        sums.append((int((v >> 32).sum()) << 32) + int((v & 0xFFFFFFFF).sum()))
        counts.append(int(counted[row].sum(dtype=np.int64)))
    return sums, counts


def planes(idx: np.ndarray):
    """24-bit indices [C][T] -> (tl uint16, th uint8)"""
    idx = np.asarray(idx, np.uint32)
    return (idx & 0xFFFF).astype(np.uint16), (idx >> 16).astype(np.uint8)


def rows_of(idx, tbook, book, d2b) -> np.ndarray:
    """the Form D tensor [C][T][9] the planes stand for"""
    return decode(tbook, book, d2b)[np.asarray(idx, np.int64)]


def stream_chunks(C: int, T: int) -> int:
    """windows apo_score_host_tuples cuts the rows into: Tc = floor(256 MiB / 3C) rounded down to the tile, >= one tile"""
    Tc = max(TILE, (256 << 20) // (3 * C) // TILE * TILE)
    Tc = min(Tc, -(-max(T, 1) // TILE) * TILE)
    return -(-T // Tc)


# ------------------------------------------------------------------------------------------------ index planes
def uniform(n, C, T, seed=0):
    return np.random.default_rng(seed).integers(0, n, (C, T), dtype=np.int64).astype(np.uint32)


def hi_byte_groups(n, C, T, seed=0):
    """every group of 8 evaluations (t // 8) carries 8 different high bytes (when n spans >= 8 of them), one per position
    q = t % 8, rotating with the group and the row; low 16 bits mixed from (c, t)"""
    nh = ((n - 1) >> 16) + 1
    t = np.arange(T, dtype=np.int64)
    out = np.empty((C, T), np.uint32)
    for c in range(C):
        h = ((t // 8) * 37 + c * 11 + seed + t % 8) % nh
        lo = (t * 40503 + c * 7919 + seed * 12345) & 0xFFFF
        idx = (h << 16) | lo
        over = idx >= n                             # only in the last, partial high plane
        idx[over] = (h[over] << 16) | (lo[over] % max(1, n & 0xFFFF))
        out[c] = idx
    return out


def boundary_indices(n):
    """0, hot - 1, hot, n - 1: those inside the dictionary"""
    return sorted({i for i in (0, hot(n) - 1, hot(n), n - 1) if 0 <= i < n})


def boundary_positions(T):
    return sorted({p for p in (0, 1, 2, 3, 7, 8, 9, TILE - 1, TILE, TILE + 1, T - 9, T - 8, T - 2, T - 1) if 0 <= p < T})


def boundary(n, C, T, seed=0):
    """uniform background; boundary_indices(n) cycle over boundary_positions(T) of every row (shifted by the row)"""
    idx = uniform(n, C, T, seed)
    special = boundary_indices(n)
    for c in range(C):
        for k, p in enumerate(boundary_positions(T)):
            idx[c, p] = special[(k + c) % len(special)]
    return idx


def warp_uniform(n, C, T, seed=0):
    """every 256-evaluation block (one warp's 32 lanes x 8) on one entry: a head entry, the last entry (the tail when n > hot),
    then a uniform block, in turn"""
    idx = uniform(n, C, T, seed)
    head, tail = min(5, n - 1), n - 1
    for c in range(C):
        for b in range(0, -(-T // 256)):
            k = (b + c) % 3
            if k < 2:
                idx[c, 256 * b:256 * (b + 1)] = (head, tail)[k]
    return idx


def reversed_freq(n, C, T, seed=0):
    """the most frequent entries at the END of the dictionary: n - 1 - geometric, so nearly every read is a tail read"""
    g = np.random.default_rng(seed).geometric(1 / 64, (C, T)) - 1
    return (n - 1 - np.minimum(g, n - 1)).astype(np.uint32)


def bank_pair(n, C, T, seed=0):
    """the lanes of a warp read different entries congruent mod 16 (the same shared-memory bank pair); the residue changes
    every 256 evaluations"""
    rng = np.random.default_rng(seed)
    t = np.arange(T, dtype=np.int64)
    out = np.empty((C, T), np.uint32)
    for c in range(C):
        r = (t // 256 + c) % 16 % n
        k = rng.integers(0, 1 << 30, T) % ((n - 1 - r) // 16 + 1)
        out[c] = r + 16 * k
    return out


PLANES = {"uniform": uniform, "hi_byte_groups": hi_byte_groups, "boundary": boundary, "warp_uniform": warp_uniform,
          "reversed_freq": reversed_freq, "bank_pair": bank_pair}


def max_groups(n, C, T, places=None, seed=0):
    """groups of 8 (t // 8) in turn: 8 x pmax, 8 x nmax, 7 x nmax + a null, 6 x nmax6 + zw + null, uniform; needs the GOOD
    entries placed (default_places).  With 8 maximal entries a group's value sum sits next to the count field of K1t."""
    p = default_places(n) if places is None else places
    idx = uniform(n, C, T, seed)
    t = np.arange(T)
    for c in range(C):
        g, q = t // 8 + c, t % 8
        kind = g % 5
        row = idx[c]
        row[kind == 0] = p["pmax"]
        row[kind == 1] = p["nmax"]
        row[kind == 2] = np.where(q[kind == 2] == (g[kind == 2] // 5) % 8, p["null"], p["nmax"])
        k3 = kind == 3
        row[k3] = np.select([q[k3] == (g[k3] // 5) % 8, q[k3] == (g[k3] // 5 + 3) % 8], [p["zw"], p["null"]], p["nmax6"])
    return idx
