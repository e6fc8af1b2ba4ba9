"""Long scoring sessions that reach the widths of the engine's integer words, and the exact arithmetic they are checked against.

Sessions (apo_score_begin / apo_score_accumulate / apo_score_finish) and the host-streaming calls add into the same words
launch after launch.  Two kinds of word could wrap there before the sums they hold reach any promised limit:

- the group words (csrc/apo_cand.cu k_cand_groups) as they were kept before: word 0 summed the low 32-bit halves and word 1
  the high halves of the two's complement of every term x = rint(fr * 2^52), word 2 took -2^64 per negative term, and nothing
  carried out of words 0 and 1.  A negative term adds about 2^32 to word 1, which wraps after ~2^32 such terms.
  parent_group_sum restates that; the words now take each flush's signed sum in the partials' limb split (fixed_group_sum).
- the limb triples (l0, l1, l2) every flush adds warp sums of 32 unsigned 32-bit halves into (flush_acc128, add_i128): the
  candidate partials, the breakdown's dimension words, the group words and the per-candidate corpus blocks.  Every reader
  takes l0 and l1 as signed int64, so a triple is read 2^96 units off once l1 passes 2^63.  parent_limbs_read restates
  the reads after F equal flushes; limb_guard restates the host-side bound that now carries every triple (k_carry_limbs)
  before LIMB_FLUSH_MAX flushes could pass, and limb_words_max the largest l0 / l1 it allows.

The legs of tests/test_gpu_long_sessions.py:
- A (leg_a_*): one resident Form T row of 2^29 + 33 evaluations at -(2 - 2^-23) and +(2 - 2^-23) in three groups,
  accumulated 32 times: groups 0 and 1 pass the old group words' wraps, group 2 never does; checked after 8 and 32.
- B (leg_b_*): constant rows at fr = -2^-52 (x = -1) accumulated leg_b_accumulates(sm_count) times, enough to take the
  old l1 past 2^63 even when every launch flushes from its fewest warps.
- C: generator rows scored once and accumulated C_SCALE = 128 times (every sum scales by 128 exactly): 2^34 random terms
  per candidate, whose low halves pass word 0's 2^64 about twice over.

Plain helpers (no pytest fixtures, no GPU)."""
from __future__ import annotations

import math

import numpy as np

import tuple_fixtures as tf

M64 = 1 << 64
FX = 1 << 52
LANES = 32

# ------------------------------------------------------------------------------------------------ launch shapes
K1_WARPS_PER_SM = 20                 # K1 (Form D, variant 0): 20 consumer warps per CTA, one CTA per SM
K1T_WARPS_PER_SM = 32                # K1t: one 1024-thread CTA per SM
PASS_MIN_WARPS_PER_SM = 8            # a per-candidate pass under MIN_CTAS 1: one 256-thread CTA per SM
MAX_WARPS_PER_SM = 64                # 2048 resident threads: the most warps any launch flushes from per SM
CB_TILE = 1024                       # evaluations per warp tile of the per-candidate passes
CC_RUN_TILES = 8                     # k_cand_corpus's run limit in tiles (the shortest of any pass)
LIMB_FLUSH_MAX = (1 << 26) - 1       # apo::LIMB_FLUSH_MAX
FLUSH_ADD_MAX = LANES * (2 ** 32 - 1)   # the most one flush adds to l0 or l1 (32 lanes of unsigned 32-bit halves)
MARGIN = 1.1


def s64(v: int) -> int:
    """a 64-bit word as the readers take it: two's complement int64"""
    v %= M64
    return v - M64 if v >= 1 << 63 else v


# ------------------------------------------------------------------------------------------------ the group words
def halves(x: int) -> tuple[int, int]:
    """(low, high) 32-bit halves of the two's complement of an int64 term"""
    u = x % M64
    return u & 0xFFFFFFFF, u >> 32


def parent_group_sum(terms: dict[int, int]) -> int:
    """the sum the old k_cand_groups_report read from the words of {term: multiplicity}: word 0 and word 1 are the sums of
    the halves modulo 2^64, word 2 is -(negative terms) modulo 2^64; the report read words 0 and 1 unsigned, word 2 signed"""
    w0 = sum(n * halves(x)[0] for x, n in terms.items()) % M64
    w1 = sum(n * halves(x)[1] for x, n in terms.items()) % M64
    w2 = s64(-sum(n for x, n in terms.items() if x < 0))
    return (w2 << 64) + (w1 << 32) + w0


def fixed_group_sum(terms: dict[int, int]) -> int:
    """the sum the words hold now: exact"""
    return sum(n * x for x, n in terms.items())


def group_wraps(terms: dict[int, int]) -> bool:
    """whether the old words lost a multiple of 2^64 in word 0 or 1"""
    return (sum(n * halves(x)[0] for x, n in terms.items()) >= M64 or sum(n * halves(x)[1] for x, n in terms.items()) >= M64)


# ------------------------------------------------------------------------------------------------ the limb triples
def flush_limbs(lane_sums) -> tuple[int, int, int]:
    """flush_acc128: the three limb sums a warp adds for 32 lane accumulators holding lane_sums (128-bit signed)"""
    lo = [v % M64 for v in lane_sums]
    hi = [(v >> 64) % M64 for v in lane_sums]
    return sum(u & 0xFFFFFFFF for u in lo) % M64, sum(u >> 32 for u in lo) % M64, sum(hi) % M64


def parent_limbs_read(F: int, limbs: tuple[int, int, int]) -> int:
    """the sum a reader (limbs_to_double, the spread report) takes from a triple after F flushes of `limbs`, with no carry"""
    l0, l1, l2 = (F * v % M64 for v in limbs)
    return (s64(l2) << 64) + (s64(l1) << 32) + s64(l0)


def exact_limbs(F: int, limbs: tuple[int, int, int]) -> int:
    l0, l1, l2 = limbs
    return F * (l0 + (l1 << 32) + (s64(l2) << 64))


def l1_wrap_flushes(limbs: tuple[int, int, int]) -> int:
    """the fewest equal flushes after which l1 reads negative"""
    return -(-(1 << 63) // limbs[1])


X_ONE = -1                                        # leg B's term: fr = -2^-52
LIMBS_ONE = flush_limbs([X_ONE] * LANES)          # every lane of a flushing warp holds at least one term (full tiles)


def limb_flush_bound(count: int, sm_count: int) -> int:
    """apo::limb_flush_bound: the most flushes one launch over `count` evaluations per candidate adds into one triple"""
    return MAX_WARPS_PER_SM * sm_count + (-(-count // CB_TILE)) // CC_RUN_TILES + 1


def limb_guard(counts, sm_count: int) -> tuple[int, int]:
    """(carries, largest flush bound between carries) of the host-side guard over launches of counts[i] evaluations"""
    since, carries, worst = 0, 0, 0
    for n in counts:
        b = limb_flush_bound(n, sm_count)
        if since + b > LIMB_FLUSH_MAX:
            carries, since = carries + 1, 0
        since += b
        worst = max(worst, since)
    return carries, worst


def limb_words_max(flushes: int) -> int:
    """the largest l0 / l1 after a carry (< 2^32) and `flushes` flushes of at most FLUSH_ADD_MAX each"""
    return (2 ** 32 - 1) + flushes * FLUSH_ADD_MAX


# ------------------------------------------------------------------------------------------------ leg A
A_T = (1 << 29) + 33
A_K = (8, 32)
A_N0 = 3 * A_T // 8
A_N1 = 3 * A_T // 8
A_N2 = A_T - A_N0 - A_N1
A_G = 3
A_TALLY_AT = 5                                     # the one evaluation whose entry also carries d0 = -1 (a 'bad' tally)
# dictionary: 0 = -(2 - 2^-23) alone on d8, 1 = +(2 - 2^-23) alone on d8, 2 = d0 = -1 (code 0 of coded dimension 0) and d8
A_ENTRIES = [tf.ENTRIES["nmax"], tf.ENTRIES["pmax"], (tf.pack_pc({0: 0, 7: 12}), tf.D2_ABSENT)]


def leg_a_dictionary():
    pc = np.array([e[0] for e in A_ENTRIES], np.uint32)
    pd = np.array([e[1] for e in A_ENTRIES], np.uint16)
    return pc, pd


def leg_a_counts() -> list[dict[int, int]]:
    """{entry: evaluations} of each group in one window"""
    g0 = {0: A_N0 - 1, 2: 1}
    g1 = {1: A_N1}
    g2 = {1: (A_N2 + 1) // 2, 0: A_N2 // 2}
    return [g0, g1, g2]


def leg_a_planes():
    """(tl, th) [1][A_T]: group 0 entry 0 (entry 2 at A_TALLY_AT), group 1 entry 1, group 2 alternating 1, 0, ..."""
    idx = np.zeros(A_T, np.uint8)
    idx[A_N0:A_N0 + A_N1] = 1
    idx[A_N0 + A_N1::2] = 1
    idx[A_TALLY_AT] = 2
    return idx.astype(np.uint16)[None], np.zeros((1, A_T), np.uint8)


def leg_a_labels() -> np.ndarray:
    labels = np.full(A_T, 2, np.uint8)
    labels[:A_N0] = 0
    labels[A_N0:A_N0 + A_N1] = 1
    return labels


def leg_a_group_terms(fx, k: int) -> list[dict[int, int]]:
    """{term: multiplicity} of each group after k accumulates, fx[i] the term of entry i"""
    return [{int(fx[e]): k * n for e, n in g.items()} for g in leg_a_counts()]


# ------------------------------------------------------------------------------------------------ leg B
B_T = (1 << 22) + 5


def leg_b_accumulates(sm_count: int, min_warps_per_sm: int = PASS_MIN_WARPS_PER_SM, margin: float = MARGIN) -> int:
    """accumulates of a B_T window after which the old l1 of every triple of the leg has passed 2^63, even if every launch
    flushed into the candidate from only min_warps_per_sm warps per SM, times the margin"""
    return math.ceil(l1_wrap_flushes(LIMBS_ONE) / (min_warps_per_sm * sm_count) * margin)


def leg_b_first_checkpoint(sm_count: int) -> int:
    """an accumulate count before any launch shape could have taken the old l1 past 2^63 (every launch at its most warps)"""
    return l1_wrap_flushes(LIMBS_ONE) // (MAX_WARPS_PER_SM * sm_count) * 5 // 8


def leg_b_checkpoints(sm_count: int) -> tuple[int, ...]:
    n = leg_b_accumulates(sm_count)
    return (leg_b_first_checkpoint(sm_count), n // 2, n)


# ------------------------------------------------------------------------------------------------ leg C
C_SCALE = 128
C_T_WIDE = (1 << 27) + 9


def leg_c_group_terms_wrap(n_terms: int, mean_low_half: float = 2.0 ** 31) -> bool:
    """whether C_SCALE accumulates of n_terms terms with random low halves (mean 2^31) pass word 0's 2^64 (in expectation)"""
    return C_SCALE * n_terms * mean_low_half >= M64
