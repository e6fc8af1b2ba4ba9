"""numpy model of the Form T copy's per-row dictionary counts (csrc/apo_kernels.h KhParams, built by build_twin_h) and of
the sum K1h takes from them.  A row's pairs are the dictionary entries its evaluations t < T name, ascending, each packed as
entry | count << 20; off[c] is the first pair of row c, off[C] the number of pairs."""
import numpy as np

COUNT_SHIFT = 20
ENTRY_MAX = (1 << COUNT_SHIFT) - 1
VALID_SHIFT = 58                                      # table entry = value + (counted << 58), apo_kernels.h KT_VALID_SHIFT


def pairs(idx, T):
    """idx [C][pitch] dictionary indices (positions >= T are pads): (off uint64 [C + 1], pairs uint64 [nnz])"""
    rows, off = [], [0]
    for r in np.asarray(idx)[:, :T]:
        e, n = np.unique(r.astype(np.int64), return_counts=True)
        assert e.size == 0 or e[-1] <= ENTRY_MAX
        rows.append(e.astype(np.uint64) | (n.astype(np.uint64) << np.uint64(COUNT_SHIFT)))
        off.append(off[-1] + e.size)
    return np.array(off, np.uint64), (np.concatenate(rows) if rows else np.zeros(0, np.uint64))


def unpack(p):
    p = np.asarray(p, np.uint64)
    return (p & np.uint64(ENTRY_MAX)).astype(np.int64), (p >> np.uint64(COUNT_SHIFT)).astype(np.int64)


def split(v):
    """table entry -> (value, counted), as kt_split: the count field sits at bit 58, rounded to the nearest"""
    v = int(v)
    k = (v + (1 << (VALID_SHIFT - 1))) >> VALID_SHIFT
    return v - (k << VALID_SHIFT), k


def entry(value, counted):
    return int(value) + (int(counted) << VALID_SHIFT)


def count_sums(off, p, tval):
    """per row (sum count * value, sum count * counted) as exact Python ints"""
    e, n = unpack(p)
    out = []
    for c in range(len(off) - 1):
        s = k = 0
        for i in range(int(off[c]), int(off[c + 1])):
            v, f = split(tval[e[i]])
            s += int(n[i]) * v
            k += int(n[i]) * f
        out.append((s, k))
    return out


def plain_sums(idx, T, tval):
    """per row (sum of values, number counted) over the evaluations t < T, one table entry at a time"""
    out = []
    for r in np.asarray(idx)[:, :T]:
        s = k = 0
        for i in r:
            v, f = split(tval[int(i)])
            s += v
            k += f
        out.append((s, k))
    return out
