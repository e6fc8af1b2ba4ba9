"""CPU model of the Form T copy's per-row dictionary counts (tests/count_model.py): the pair layout (packing, order, offsets,
pads left out), and that sum count * value equals the per-evaluation sum exactly, at the value, entry and row-length edges.
No GPU needed."""
import numpy as np
import pytest

import count_model as cm

VMAX = (1 << 53) - 1


def table(values_flags):
    """an entry-order table with the zero sentinel after the last entry"""
    return [cm.entry(v, f) for v, f in values_flags] + [0]


def padded(idx, pitch, pad=0xFFFFFF):
    out = np.full((len(idx), pitch), pad, np.int64)
    for c, r in enumerate(idx):
        out[c, :len(r)] = r
    return out


def check(idx, T, tval):
    off, p = cm.pairs(idx, T)
    assert off[0] == 0 and off[-1] == len(p)
    e, n = cm.unpack(p)
    for c in range(len(off) - 1):
        seg = e[int(off[c]):int(off[c + 1])]
        assert np.all(np.diff(seg) > 0)                          # ascending, each entry once
        assert int(n[int(off[c]):int(off[c + 1])].sum()) == T      # every evaluation t < T counted once, no pad
    assert cm.count_sums(off, p, tval) == cm.plain_sums(idx, T, tval)
    return off, p


def test_packing():
    off, p = cm.pairs(np.array([[3, 3, 1, cm.ENTRY_MAX, 3]]), 5)
    assert list(off) == [0, 3]
    assert [int(x) for x in p] == [1 | (1 << 20), 3 | (3 << 20), cm.ENTRY_MAX | (1 << 20)]


@pytest.mark.parametrize("flags", [(1, 1), (0, 0), (1, 0)])
def test_extreme_values(flags):
    """entries at +-(2^53 - 1), counted or not, repeated so that count * value passes 2^64"""
    tval = table([(VMAX, flags[0]), (-VMAX, flags[1]), (1, 1), (-1, 0)])
    T = 3000
    rng = np.random.default_rng(1)
    idx = rng.integers(0, 4, (3, T))
    idx[1] = 0                                                   # one entry repeated T times
    idx[2, : T // 2] = 1
    off, p = check(idx, T, tval)
    s, k = cm.count_sums(off, p, tval)[1]
    assert s == T * VMAX and k == T * flags[0]
    big = [(VMAX, 1)] * 2
    assert cm.count_sums(*cm.pairs(np.zeros((1, 1 << 13), np.int64), 1 << 13), table(big))[0][0] == (1 << 13) * VMAX


def test_null_row():
    """a row of null entries (value 0, not counted) only"""
    tval = table([(0, 0), (5, 1)])
    idx = np.array([[0] * 100, [0, 1] * 50])
    off, p = check(idx, 100, tval)
    assert cm.count_sums(off, p, tval)[0] == (0, 0)


def test_entry_edges():
    """entries >= 2^16, in [end, 2^16) (without a K1t2 slot), and the largest the packing holds"""
    n = cm.ENTRY_MAX + 1
    rng = np.random.default_rng(2)
    vals = rng.integers(-VMAX, VMAX, n + 1)
    vals[[65535, 65536, n - 1]] = [VMAX, -VMAX, VMAX]
    flags = rng.integers(0, 2, n + 1)
    tval = [cm.entry(v, f) for v, f in zip(vals, flags)]
    tval[n] = 0
    T = 5000
    idx = rng.integers(0, 4000, (4, T))
    idx[0, :6] = [65535, 65536, 65535 - 15 * 512, 65535 - 15 * 512 - 1, n - 1, n - 1]
    idx[1, 100:200] = rng.integers(65536, n, 100)
    idx[3] = n - 1
    check(idx, T, tval)


@pytest.mark.parametrize("T", [1, 7, 8, 63, 64, 65, 1001])
def test_ragged_rows_leave_out_pads(T):
    """rows padded to 64 evaluations: only t < T is counted, whatever the pads hold"""
    pitch = (T + 63) // 64 * 64
    rng = np.random.default_rng(T)
    tval = table([(int(v), int(f)) for v, f in zip(rng.integers(-VMAX, VMAX, 50), rng.integers(0, 2, 50))])
    idx = padded([rng.integers(0, 50, T) for _ in range(5)], pitch, pad=49)
    off, p = check(idx, T, tval)
    assert np.array_equal(off, cm.pairs(idx[:, :T], T)[0])
