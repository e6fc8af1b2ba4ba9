"""numpy model of the exception list of the Form T copy and of K1t2's correction (no GPU needed).

The copy keeps every evaluation's dictionary index as a 16-bit plane tl and an 8-bit plane th.  K1t2 reads tl alone and
adds table[tl]; the evaluations with th != 0 (exceptions) are listed per row as {position, full index}, sorted by
position, with a block index xb[c][b] = list offset of row c's first exception at or after position 8192 b (b = nblk ends
the row).  A CTA corrects the exceptions of each (candidate, tile range) segment it streamed: it reads xb at the blocks
holding the segment's ends, skips the exceptions outside the segment, and adds table[full] - table[full & 0xFFFF], value
and count split, the count as a signed quantity.  The model checks that this equals the sum over the full indices for
windows and CTA cuts inside and across blocks."""
import numpy as np

XBLOCK = 8192
TILE = 16384
SHIFT = 58


def build_list(tl, th, T):
    """(xb [C][nblk + 1], xs [n][2]) as run_tx_build writes them: a count per (row, block), an exclusive scan over the
    flattened [C][nblk + 1] counts (the last column counts nothing), then the exceptions in row and position order"""
    C = tl.shape[0]
    nblk = -(-T // XBLOCK)
    counts = np.zeros((C, nblk + 1), np.int64)
    xs = []
    for c in range(C):
        pos = np.nonzero(th[c, :T])[0]
        counts[c, :nblk] = np.bincount(pos // XBLOCK, minlength=nblk)
        full = tl[c, pos].astype(np.uint32) | (th[c, pos].astype(np.uint32) << 16)
        xs.append(np.stack([pos.astype(np.uint32), full], 1))
    flat = counts.reshape(-1)
    xb = (np.cumsum(flat) - flat).reshape(C, nblk + 1).astype(np.uint32)
    return xb, np.concatenate(xs).astype(np.uint32)


def split(v):
    """table entry -> (value, count), as kt_split"""
    k = (v + (1 << (SHIFT - 1))) >> SHIFT
    return v - (k << SHIFT), k


def segment(tval, tl, xb, xs, c, lo, hi):
    """what one CTA adds for row c's absolute positions [lo, hi): the stream over tl, then the correction"""
    v, k = split(tval[tl[c, lo:hi].astype(np.int64)])
    val, cnt = int(v.sum()), int(k.sum())
    x0, x1 = int(xb[c, lo // XBLOCK]), int(xb[c, (hi - 1) // XBLOCK + 1])
    dcnt = 0
    for pos, full in xs[x0:x1]:
        if lo <= pos < hi:
            vf, kf = split(int(tval[full]))
            vl, kl = split(int(tval[full & 0xFFFF]))
            val += vf - vl
            dcnt += kf - kl
    return val, cnt + dcnt, dcnt


def planes(seed, C, T, n_tuples):
    rng = np.random.default_rng(seed)
    idx = rng.integers(0, 1 << 16, (C, T)).astype(np.uint32)
    rare = rng.random((C, T)) < 0.01
    idx[rare] = rng.integers(1 << 16, n_tuples, int(rare.sum()))
    idx[1] = rng.integers(0, 1 << 16, T)                             # a row without exceptions
    idx[2] = rng.integers(1 << 16, n_tuples, T)                      # a row of exceptions only
    idx[3, XBLOCK:2 * XBLOCK] = rng.integers(1 << 16, n_tuples, XBLOCK)   # a block of exceptions
    idx[0, 0] = idx[0, T - 1] = n_tuples - 1                         # at the first and the last position
    return idx, (idx & 0xFFFF).astype(np.uint16), (idx >> 16).astype(np.uint8)


def table(seed, n):
    """entries rint(x * 2^52) + (counted << 58); the high entries are mostly uncounted, the low ones counted, so the
    correction's net count is negative"""
    rng = np.random.default_rng(seed)
    fx = rng.integers(-(1 << 40), 1 << 40, n)
    counted = np.where(np.arange(n) < (1 << 16), rng.random(n) < 0.95, rng.random(n) < 0.1)
    return fx + (counted.astype(np.int64) << SHIFT)


def test_list_layout():
    C, T, n = 5, 3 * XBLOCK + 1001, 200_000
    idx, tl, th = planes(7, C, T, n)
    xb, xs = build_list(tl, th, T)
    nblk = xb.shape[1] - 1
    assert xb[0, 0] == 0 and xb[C - 1, nblk] == len(xs)
    assert all(xb[c, nblk] == xb[c + 1, 0] for c in range(C - 1))  # the end of row c starts row c + 1
    assert xb[1, 0] == xb[1, nblk]                                  # no exceptions
    assert xb[2, nblk] - xb[2, 0] == T                              # only exceptions
    assert xb[3, 2] - xb[3, 1] == XBLOCK
    row0 = xs[xb[0, 0]:xb[0, nblk]]
    assert row0[0, 0] == 0 and row0[-1, 0] == T - 1 and row0[0, 1] == n - 1
    for c in range(C):
        r = xs[xb[c, 0]:xb[c, nblk]]
        assert np.all(np.diff(r[:, 0].astype(np.int64)) > 0)
        assert np.array_equal(r[:, 1], idx[c, r[:, 0]])
        for b in range(nblk):                                        # xb[c][b]: first exception at or after 8192 b
            assert np.all(xs[xb[c, 0]:xb[c, b], 0] < b * XBLOCK)
            assert np.all(xs[xb[c, b]:xb[c, nblk], 0] >= b * XBLOCK)


def test_correction_equals_the_full_indices():
    C, T, n = 5, 3 * XBLOCK + 1001, 200_000
    idx, tl, th = planes(11, C, T, n)
    tval = table(12, n + 1)
    xb, xs = build_list(tl, th, T)
    negative = False
    windows = ((0, T), (8, XBLOCK - 8), (XBLOCK, XBLOCK), (XBLOCK + 8, 2 * XBLOCK), (T - 1, T), (0, 1), (4096, T - 3))
    for first, end in windows:
        for c in range(C):
            v, k = split(tval[idx[c, first:end].astype(np.int64)])
            want = (int(v.sum()), int(k.sum()))
            assert segment(tval, tl, xb, xs, c, first, end)[:2] == want, (first, end, c)
            # the window cut into CTA segments at tile edges relative to the window (and one cut off the block grid)
            cuts = sorted({first, end} | {min(end, first + t) for t in range(TILE, end - first, TILE)} | {min(end, first + 5000)})
            got = [segment(tval, tl, xb, xs, c, a, b) for a, b in zip(cuts, cuts[1:])]
            assert (sum(g[0] for g in got), sum(g[1] for g in got)) == want, (first, end, c)
            negative |= any(g[2] < 0 for g in got)
    assert negative                                                  # the signed count path was exercised
