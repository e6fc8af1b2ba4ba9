"""Hand-built Form D tensors that reach the edges of K1 / K1r / K1q (csrc/apo_kernels.cu, csrc/apo_compact.cu) and of the K3
tail (csrc/apo_corpus.cuh finalize_block), and the plain references they are checked against.

- Shapes: the tile of every kernel variant (TILES_K1, TILES_KQ), rows of T = TILE - 8 ... 2 TILE + 1 around it (t_edges),
  windows whose start is off the tile grid, and short rows (T < 8) with many candidates, so that one CTA's tile range crosses
  dozens of candidates and flushes on every change (shape_dims, short_dims).
- Extremes: evaluations with every dimension at +-MAXF = 511.99997 (the largest fp32 below 512), all one sign or
  alternating, whose sums pass 2^64, 2^72 and ~2^83 (extreme_dims, huge_dims); and candidates whose exact sum S lands on a
  binary64 tie, with and without a sticky bit below it, in both branches of limbs_to_double (TIE_SUMS, tie_dims).
- Score keys: candidates whose binary64 scores share their top 7 ... 1 bytes, all-equal rows, tie groups, -inf rows
  (count 0) (key_dims).

Exact sums are built from single-dimension evaluations of value +-2^e (pow2_rows): (v * w) / w == v exactly for a power
of two v, so such an evaluation adds exactly +-2^(e + 52) to the fixed-point sum; a value 0.0 adds 0 and is counted, an
all-NaN row is not counted.  Every target the GPU tests use is nevertheless the oracle's (oracle.score_dims_fx /
score_records_fx); scores come from sharding.scores_from_partials (Python's correctly rounded int -> float), top-K from
sharding.topk_indices.  fx_model restates the Form D arithmetic in numpy (binary64, no FMA) for the APO_SCORE_RECIP
variants, which the oracle does not model; on the IEEE division it is checked against the oracle.

Plain helpers, imported by the tests that use them (no fixtures, no GPU)."""
import ctypes
import importlib

import numpy as np

import oracle

sharding = importlib.import_module("senweaver-ide_b200.sharding")
engine_mod = importlib.import_module("senweaver-ide_b200.engine")

FX = 1 << 52
TILES_K1 = {0: 2560, 1: 2048, 2: 1536, 3: 1024, 4: 3072}               # K1 / K1r: 4 evaluations x consumer threads
TILES_KQ = {0: 5120, 1: 4096, 2: 3072, 3: 2560, 4: 5120, 5: 5120, 6: 5120}
MAXF = np.float32(np.nextafter(np.float32(512), np.float32(0)))       # 511.99997
NAN = np.float32("nan")
HOST_OUT_MAX = 64 << 10                                              # result blocks up to this size are written by the kernel


def t_edges(tile: int):
    """row lengths around one tile and two: the full-tile path, the partial-tile path and its pad evaluations"""
    return (tile - 8, tile - 1, tile, tile + 1, tile + 4, tile + 7, tile + 8, 2 * tile - 1, 2 * tile + 1)


def window_starts(tile: int, align: int):
    """window starts off the tile grid (multiples of `align`: 4 for Form D / R, 8 for Form Q)"""
    return (0, align, tile - align, tile + 3 * align)


# ------------------------------------------------------------------------------------------------ exact rows
def single(v, dim: int = 0) -> np.ndarray:
    row = np.full(9, NAN, np.float32)
    row[dim] = v
    return row


def pow2_rows(S: int, dim: int = 0, top: int = 60) -> list:
    """single-dimension rows whose fixed-point values (fx = v * 2^52) sum to exactly S: 2^top per row for the bulk, then one
    row per set bit of the remainder"""
    sign = -1.0 if S < 0 else 1.0
    q, r = divmod(abs(S), 1 << top)
    rows = [single(np.float32(sign * 2.0 ** (top - 52)), dim)] * q
    rows += [single(np.float32(sign * 2.0 ** (b - 52)), dim) for b in range(top) if (r >> b) & 1]
    return rows


def candidate(S: int, n: int, T: int, dim: int = 0) -> np.ndarray:
    """[T][9]: rows summing to S, padded with counted zeros to n evaluations, then with not-counted all-NaN rows to T"""
    rows = pow2_rows(S, dim)
    assert len(rows) <= n <= T, (S, n, T)
    rows += [single(np.float32(0.0), dim)] * (n - len(rows))
    rows += [np.full(9, NAN, np.float32)] * (T - n)
    return np.stack(rows) if rows else np.zeros((0, 9), np.float32)


# ------------------------------------------------------------------------------------------------ references
def oracle_fx(dims: np.ndarray, w=None):
    return oracle.score_dims_fx(np.ascontiguousarray(dims, np.float32), w=w)


def fx_model(dims: np.ndarray, w=None, recip: bool = False, chunk: int = 1 << 20):
    """per-candidate (sums, counts) of Form D dims [C][T][9]: weighted sum in push order, total weight of the present
    weights in push order, ws / tw (or ws * RN(1/tw) with recip), rint(fr * 2^52); exact Python-int sums"""
    w = oracle.weights() if w is None else np.asarray(w, np.float64)
    dims = np.asarray(dims, np.float32)
    sums, counts = [], []
    for row in dims:
        s, n = 0, 0
        for a in range(0, len(row), chunk):
            d = row[a:a + chunk].astype(np.float64)
            p = ~np.isnan(d)
            g = np.where(p, d, 0.0)
            ws = np.zeros(len(d))
            tw = np.zeros(len(d))
            for i in range(9):
                ws = ws + g[:, i] * w[i]
                tw = tw + np.where(p[:, i], w[i], 0.0)
            ok = tw > 0
            with np.errstate(divide="ignore", invalid="ignore"):
                fr = ws * (1.0 / tw) if recip else ws / tw
            fx = np.rint(np.where(ok, fr, 0.0) * float(FX)).astype(np.int64)
            s += (int((fx >> 32).sum()) << 32) + int((fx & 0xFFFFFFFF).sum())
            n += int(ok.sum())
        sums.append(s)
        counts.append(n)
    return sums, counts


def scores_of(sums, counts) -> np.ndarray:
    return sharding.scores_from_partials(sums, counts)


# ------------------------------------------------------------------------------------------------ shapes
def shape_dims(C: int, T: int, seed: int = 0) -> np.ndarray:
    """generator rows (categorical: Form Q can hold them) with every 7th row at +MAXF in all dimensions, every 11th at -MAXF,
    every 13th all-NaN, and runs of 4 aligned +MAXF rows (one consumer thread's four pre-added terms at the int64 edge)"""
    d = oracle.gen_dims(0x5EED0000 + seed, 0, C, 0, T, 300, 8)
    t = np.arange(T)
    for c in range(C):
        d[c, (t + c) % 7 == 3] = MAXF
        d[c, (t + 2 * c) % 11 == 5] = -MAXF
        d[c, (t + c) % 13 == 0] = NAN
        d[c, ((t // 4) + c) % 97 == 1] = MAXF
    return d


def short_dims(C: int, T: int, seed: int = 0) -> np.ndarray:
    """many candidates with rows shorter than 8: one tile per candidate, CTA ranges cross dozens of candidates"""
    return shape_dims(C, T, seed)


def shape_records(C: int, T: int, seed: int = 0) -> np.ndarray:
    return oracle.gen_records(0x5EED1000 + seed, oracle.STREAM_ROLLOUT, 0, C, 0, T, 300, 8)


# ------------------------------------------------------------------------------------------------ extremes
def extreme_dims(T: int = 2 * 1024 + 9) -> np.ndarray:
    """[5][T][9]: all +MAXF (sum passes 2^72 at T >= 2057), all -MAXF, alternating +-MAXF (the low limb wraps at every
    step: carries and borrows into the upper limbs), 9 x +MAXF then nothing counted (passes 2^64), pairs of equal sign"""
    d = np.full((5, T, 9), MAXF, np.float32)
    d[1] = -MAXF
    sgn = np.where(np.arange(T) % 2 == 0, 1, -1).astype(np.float32)
    d[2] *= sgn[:, None]
    d[3, 9:] = NAN
    d[4] *= np.where(np.arange(T) // 2 % 2 == 0, 1, -1).astype(np.float32)[:, None]
    return d


def huge_dims(T: int = (1 << 22) + 5) -> np.ndarray:
    """[2][T][9]: all +MAXF and all -MAXF over 2^22 + 5 evaluations: sums just past +-2^83"""
    d = np.full((2, T, 9), MAXF, np.float32)
    d[1] = -MAXF
    return d


# S (in 2^-52 units) -> what float(S) must be: ties-to-even at 2^53 + 1 / 2^53 + 3 (hi == 0 branch, u64 -> binary64), and in
# the 128-bit branch at 2^65 + 2^12 (tie, even is down) and 2^65 + 3 * 2^12 (tie, even is up), with a sticky bit one below
# the cut (2^65 + 2^12 + 1: must round up), far below it (2^70 + 2^17 + 1, shift 7), or one short of the tie
TIE_SUMS = (
    (1 << 53) + 1, (1 << 53) + 3, (1 << 54) + 2, (1 << 54) + 6, (1 << 54) + 3,
    (1 << 65) + (1 << 12), (1 << 65) + (1 << 12) + 1, (1 << 65) + 3 * (1 << 12), (1 << 65) + (1 << 12) - 1,
    (1 << 70) + (1 << 17), (1 << 70) + (1 << 17) + 1,
)
TIE_N = 2048                     # evaluations per tie candidate (a power of two: score = float(S) / 2^52 / n exactly)


def tie_sums():
    """TIE_SUMS and their negative mirrors"""
    return [s for S in TIE_SUMS for s in (S, -S)]


def tie_dims() -> np.ndarray:
    sums = tie_sums()
    return np.stack([candidate(S, TIE_N, TIE_N, dim=k % 9) for k, S in enumerate(sums)])


def is_binary64_tie(S: int) -> bool:
    """S lies exactly halfway between two neighbouring binary64 values"""
    m = abs(S)
    if m.bit_length() <= 53:
        return False
    half = 1 << (m.bit_length() - 54)
    return m % (2 * half) == half


# ------------------------------------------------------------------------------------------------ score keys
KEY_T = 16                       # evaluations per candidate row, counted ones always KEY_N (a power of two)
KEY_N = 16


def key_sum(c: int, mode: str) -> int | None:
    """exact sum of candidate c (None: no counted evaluation, score -inf).  mixed: classes by c mod 17 -- sums
    2^52 + k * 2^(8j) (scores share their top 7 - j bytes within class j), their negatives, differing exponents, 0, one
    large tie group, -inf rows; equal: every candidate the same; sparse: 3 of 4 candidates -inf"""
    h = (c * 2654435761) >> 7 & 0xFFFF
    if mode == "equal":
        return (1 << 52) + 12345
    if mode == "sparse" and c % 4:
        return None
    cls = c % 17
    if cls < 7:
        return (1 << 52) + ((h % (16 if cls == 6 else 256)) << (8 * cls))
    if cls < 14:
        j = cls - 7
        return -((1 << 52) + ((h % (16 if j == 6 else 256)) << (8 * j)))
    if cls == 14:
        return (1 if h & 1 else -1) << (40 + h % 24)
    if cls == 15:
        return (1 << 52) + 12345 if h % 3 else 0
    return None


def key_dims(C: int, mode: str = "mixed") -> np.ndarray:
    out = np.full((C, KEY_T, 9), NAN, np.float32)
    for c in range(C):
        S = key_sum(c, mode)
        if S is not None:
            out[c] = candidate(S, KEY_N, KEY_T, dim=c % 9)
    return out


def key_targets(C: int, mode: str = "mixed"):
    sums = [key_sum(c, mode) or 0 for c in range(C)]
    counts = [0 if key_sum(c, mode) is None else KEY_N for c in range(C)]
    return sums, counts


def score_key(s: float) -> int:
    """the kernel's ascending order-preserving map of a binary64 score (apo_corpus.cuh score_key)"""
    b = int(np.float64(s).view(np.uint64))
    return (~b & 0xFFFFFFFFFFFFFFFF) if b >> 63 else b | (1 << 63)


def straddling_k(scores: np.ndarray):
    """a K whose K-th and (K+1)-th best scores are equal (a tie group straddles K), nearest to the middle; None if none"""
    order = sharding.topk_indices(scores, len(scores))
    s = scores[order]
    ks = [k for k in range(1, len(s)) if s[k - 1] == s[k]]
    return min(ks, key=lambda k: abs(k - len(s) // 2)) if ks else None


def k_values(scores: np.ndarray):
    C = len(scores)
    ks = {0, 1, C}
    k = straddling_k(scores)
    if k is not None:
        ks.add(k)
    return sorted(k for k in ks if k <= C)


# ------------------------------------------------------------------------------------------------ K3 sizes
REPORT_BYTES = ctypes.sizeof(engine_mod.CorpusReport)
META_BYTES = 32


def _up16(x: int) -> int:
    return (x + 15) // 16 * 16


def result_bytes(C: int, K: int) -> int:
    """bytes of the result block (apo_abi.cu result_layout): scores | counts | top-K | report | meta"""
    return _up16(_up16(16 * C + 4 * K) + REPORT_BYTES) + META_BYTES


def host_out_edge(k_of_c) -> int:
    """the largest C whose result block (K = k_of_c(C)) the finalising kernel still writes to page-locked memory itself"""
    C = 1
    while result_bytes(C + 1, k_of_c(C + 1)) <= HOST_OUT_MAX:
        C += 1
    return C


K3_SIZES = (1, 31, 32, 33, 1023, 1024, 1025, 2047, 2048, 2049, 4096)


def k3_sizes():
    e1, ec = host_out_edge(lambda C: 1), host_out_edge(lambda C: C)
    return sorted(set(K3_SIZES) | {e1, e1 + 1, ec, ec + 1})
