"""The fixtures of tests/kh_fixtures.py reach the edges of K1h's launch they claim (no GPU): the plan model's ballot search
against bisect, the probe-offset cuts of every search round, the stream's rows at +-1 of both strides, both digest passes
in one launch with uneven and zero shares, and K3 sizes on both sides of the tail's switch to the radix select."""
import bisect

import numpy as np
import pytest

import count_model as cm
import k1_fixtures as kf
import kh_fixtures as kh

ROUNDS = {1: 0, 2: 1, 32: 1, 33: 2, 1024: 2, 1025: 3, 4097: 3}
ALL_D = (-1, 0, 1)


def plans(fx, cd_n=kh.ROW_KEYS, corpus_on=True):
    nnz = int(fx.off[-1])
    return {g: kh.kh_plan(nnz, fx.off, cd_n, g, corpus_on) for g in kh.GRIDS}


def test_search_matches_bisect_on_random_offsets():
    """runs of rows of equal length, single-pair rows, empty rows and long rows; every pair position of small arrays"""
    rng = np.random.default_rng(0x5EEDF210)
    for C in (1, 2, 3, 31, 32, 33, 63, 64, 65, 1023, 1024, 1025, 1056, 4097, 40_000):
        for kind in ("random", "runs", "empty", "skewed"):
            if kind == "random":
                ln = rng.integers(1, 50, C)
            elif kind == "runs":
                ln = np.repeat(rng.integers(1, 6, C // 7 + 1), 7)[:C]
            elif kind == "empty":
                ln = rng.integers(0, 3, C)
                ln[-1] = max(ln[-1], 1)
            else:
                ln = np.ones(C, np.int64)
                ln[rng.integers(0, C)] = 5000
            off = np.concatenate([[0], np.cumsum(ln)])
            nnz = int(off[-1])
            los = range(nnz) if nnz <= 3000 else rng.integers(0, nnz, 3000)
            for lo in los:
                row, rounds = kh.search(off, C, int(lo))        # asserts row == bisect
                assert row == bisect.bisect_right(off.tolist(), int(lo)) - 1
                assert len(rounds) <= ROUNDS.get(C, 4)


@pytest.mark.parametrize("fx", kh.search_fixtures(), ids=lambda f: f.name)
def test_search_fixture_edges(fx):
    off = fx.off
    C, nnz = len(off) - 1, int(off[-1])
    assert kh.lengths_of(off).min() >= 1 and kh.launched_grid(nnz, 13) == 13
    p = plans(fx)
    hits = set().union(*(kh.probe_hits(q, off) for q in p.values()))
    R = ROUNDS[C]
    assert max(len(c.rounds) for q in p.values() for c in q.ctas) == R
    if C == 2:
        assert {r for r, _ in hits} <= {1}
    else:
        assert hits == {(r, d) for r in range(1, R + 1) for d in ALL_D}, sorted(hits)
    for g, q in p.items():
        assert q.grid == kh.launched_grid(nnz, g)
        for cta in q.ctas:                                          # the segments tile the CTA's range
            assert sum(t - s for _, s, t in cta.segs) == cta.hi - cta.lo
    if fx.name in ("c1", "c2_spans"):
        assert all(cta.segs[0][0] == 0 for q in p.values() for cta in q.ctas)        # one row under every CTA
    if fx.name in ("c32", "c33", "c1024", "c1025"):
        last = int(off[C - 1])
        inside = [(g, c.k) for g, q in p.items() for c in q.ctas[1:] if c.lo > last + 1]
        assert inside and p[None].ctas[-1].row == C - 1, fx.name
    if C == 4097:
        assert p[None].grid == kh.H100_SMS                         # the default grid, not one the pairs cap
    print(fx.name, "C", C, "rounds", R, "probe hits (round, d)", sorted(hits))


def test_stride_rows():
    whole, mid = kh.stride_fixtures()
    lw = kh.lengths_of(whole.off)
    assert set(kh.STRIDE_ROWS) <= set(lw.tolist())
    for corpus_on, nt, stride in ((True, kh.NT_WARP, kh.STRIDE_WARP), (False, kh.KH_THREADS, kh.STRIDE_BLOCK)):
        q = kh.kh_plan(int(whole.off[-1]), whole.off, 0, 2, corpus_on)
        assert {c.nt for c in q.ctas} == {nt}
        segs = [t - s for c in q.ctas for _, s, t in c.segs if t - s in kh.STRIDE_ROWS]
        assert sorted(segs) == sorted(kh.STRIDE_ROWS)                 # every stride row whole inside one CTA
        got = sorted({n % stride for n in segs})
        assert {0, 1, stride - 1} <= set(got), got
        print("whole rows at 2 CTAs, NT", nt, "lengths mod", stride, got)
    for corpus_on in (True, False):
        q = kh.kh_plan(int(mid.off[-1]), mid.off, 0, kh.MID_GRID, corpus_on)
        started = []
        for cta in q.ctas[1:]:
            c, s, t = cta.segs[0]
            assert s == cta.lo > int(mid.off[c])                       # the CTA starts inside the row
            started.append(t - s)
        assert started == list(kh.STRIDE_MID)
    print("rows started mid-CTA at 7 CTAs: pairs left", list(kh.STRIDE_MID),
          "mod 7936", [n % kh.STRIDE_WARP for n in kh.STRIDE_MID], "mod 8192", [n % kh.STRIDE_BLOCK for n in kh.STRIDE_MID])


def test_digest_passes():
    seen = {"mixed": 0, "uneven": 0, "zero": 0}
    deltas = set()
    for fx in kh.digest_fixtures():
        nnz = int(fx.off[-1])
        for n in kh.DIG_KEYS:
            q = kh.kh_plan(nnz, fx.off, n, kh.DIG_GRID)
            assert q.grid == kh.DIG_GRID and sum(c.share for c in q.ctas) == n
            blocks = {c.block for c in q.ctas}
            seen["mixed"] += blocks == {True, False}
            seen["uneven"] += n % kh.DIG_GRID in (1, 6) and len({c.share for c in q.ctas}) == 2
            seen["zero"] += any(c.share == 0 for c in q.ctas)
            for c in q.ctas:
                if c.share:
                    deltas.add(c.hi - c.lo - kh.KH_PAIRS_PER_ENTRY * c.share)
                assert c.block == (c.hi - c.lo < kh.KH_PAIRS_PER_ENTRY * c.share)
                assert c.nt == (kh.KH_THREADS if c.block else kh.NT_WARP)
            print(fx.name, "n", n, [(c.hi - c.lo, c.share, "block" if c.block else "warp") for c in q.ctas])
    assert seen["mixed"] >= 3 and seen["uneven"] >= 4 and seen["zero"] >= 4, seen
    assert {-1, 0, 1} <= deltas, deltas


def test_row_fixtures_keep_their_counts():
    """the counts are held (8 nnz <= C T / 2), the pool covers every row, and the rows' distinct evaluations are exactly
    the offsets (count_model on the pool indices of a smaller fixture)"""
    for fx in kh.search_fixtures() + kh.stride_fixtures() + kh.digest_fixtures():
        ln = kh.lengths_of(fx.off)
        T = kh.gate_T(fx.off)
        assert 16 * int(ln.sum()) <= len(ln) * T and ln.max() <= kh.POOL_N
    fx = kh.search_fixtures()[3]                                        # C = 32
    dims = kh.fixture_dims(fx)
    u = np.unique(dims.view(np.uint32).reshape(-1, 9), axis=0, return_inverse=True)[1].reshape(dims.shape[:2])
    off, _ = cm.pairs(u, dims.shape[1])
    assert np.array_equal(off.astype(np.int64), fx.off)


def test_k3_cases():
    sizes = {C for C, _ in kh.k3_cases()}
    assert {1024, 1025} <= sizes and kh.tail_select(1024) == "rank" and kh.tail_select(1025) == "radix"
    for C, mode in kh.k3_cases():
        off = kh.k3_offsets(C, mode)
        assert 16 * int(off[-1]) <= C * kh.K3_T
        if C in kh.K3_ALL_MODES or C in (1024, 1025):
            fx, n = kf.oracle_fx(kh.k3_dims(C, mode))
            s = kf.scores_of(fx, n)
            if mode != "equal" and C > 17:
                assert kf.straddling_k(s) is not None                     # a K inside a tie group
                assert np.isneginf(s).any()
            assert len(kf.k_values(s)) >= (3 if C > 1 else 2)
