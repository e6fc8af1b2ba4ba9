"""CPU model of K1t2's slot layout (tests/slot_model.py): the slot-order table and the slot plane give every row the sum the
plain gather of the entry-order table gives, at the layout's edges; the copies a half-warp instruction names keep clear of
each other; and the wavefront model sees fewer conflicts than the plain index plane.  No GPU needed."""
import numpy as np
import pytest

import slot_model as sm


def table(n, seed):
    rng = np.random.default_rng(seed)
    v = rng.integers(-(1 << 52), 1 << 52, n + 1, dtype=np.int64) + (rng.integers(0, 2, n + 1, dtype=np.int64) << 58)
    v[n] = 0
    return v


def skewed(C, T, n, seed, a=1.3):
    rng = np.random.default_rng(seed)
    idx = (rng.zipf(a, (C, T)) - 1) % n
    return idx.astype(np.int64)


def plain(idx, tval):
    return tval[idx].sum(axis=1, dtype=np.int64)


@pytest.mark.parametrize("n,h", [(1, 1), (600, 512), (70000, 512), (70000, 256), (70000, 0), (1 << 20, 512)])
def test_slot_table_names_each_entry(n, h):
    h = min(h, n)
    tval = table(n, n + h)
    end = sm.slot_end(n, h)
    sval = sm.slot_table(tval, h, end)
    assert len(sval) == end + 15 * h + 1 <= 65536
    for e in (0, h - 1, h, end - 1):
        if 0 <= e < n:
            slots = [16 * e + k for k in range(16)] if e < h else [e + 15 * h + 1]
            assert all(sval[s] == tval[e] for s in slots), e
    assert sval[16 * h] == 0


@pytest.mark.parametrize("T", [1, 127, 128, 1000, 4099])
@pytest.mark.parametrize("n,h", [(300, 512), (70000, 512), (200000, 512), (70000, 0)])
def test_slot_plane_sums_equal_plain_gather(T, n, h):
    h = min(h, n)                                                # as build_twin_t2: no more replicated entries than entries
    idx = skewed(3, T, n, T + n)
    idx[0, :min(T, 4)] = [h - 1, h, sm.slot_end(n, h) - 1, min(n - 1, 65535)][:min(T, 4)]   # the edges of the layout
    if n > 65536:
        idx[1, -1] = n - 1                                       # an exception
    idx = np.clip(idx, 0, n - 1)
    tval = table(n, 7)
    end = sm.slot_end(n, h)
    slots = sm.slot_plane(idx, h, end)
    assert slots.shape == idx.shape
    assert np.array_equal(sm.row_sums(idx, slots, tval, h, end), plain(idx, tval))
    # every slot names its evaluation's entry, or the zero slot for a listed one
    sval = sm.slot_table(tval, h, end)
    listed = idx >= end
    assert np.array_equal(sval[slots.astype(np.int64)][~listed], tval[idx][~listed])
    assert np.all(slots[listed] == 16 * h)


def test_half_warp_copies_keep_clear():
    """in a half-warp instruction, distinct hot entries never share a bank pair while a free one is left"""
    idx = skewed(2, 4096, 70000, 3)
    h, end = 512, sm.slot_end(70000, 512)
    slots = sm.slot_plane(idx, h, end).astype(np.int64)
    g = slots.reshape(2, 32, 16, 8).transpose(0, 1, 3, 2).reshape(-1, 16)
    for row in g:
        cold = row[row >= 16 * h]
        hot = np.unique(row[row < 16 * h])
        pairs = hot & 15
        if len(np.unique(cold & 15)) + len(hot) <= 16:
            assert len(np.unique(pairs)) == len(hot)
            assert not set(pairs) & set(cold & 15)


def test_choose_h_keeps_the_second_list_short():
    n, N = 65536, 65536 * 64
    counts = np.full(n, 64)                                      # 2^16 equally frequent entries
    h, end = sm.choose_h(counts, N)
    assert int(counts[end:].sum()) * 64 <= N
    assert h < 512
    counts = np.sort(np.random.default_rng(1).zipf(1.5, 200000))[::-1]
    h, end = sm.choose_h(counts, int(counts.sum()))
    assert h == 512 and end == 65535 - 15 * 512


def test_wavefront_model_favours_slots():
    n = 200000
    idx = skewed(4, 1 << 15, n, 5, a=1.2)
    h, end = 512, sm.slot_end(n, 512)
    new = sm.wavefronts(sm.slot_plane(idx, h, end))
    old = sm.wavefronts(idx & 0xFFFF, hot=24576)
    assert 2.0 <= new["warp"] < old["warp"]
    assert new["half_warps"] < old["half_warps"]
