"""The Form T builders of tuple_fixtures.py deliver what they claim, checked on the CPU: the byte layout of the index planes,
where the boundary indices land, distinct entries, no power-of-two period in the entry values, a lossless decode, and the
reference integers of small cases worked out from the per-entry values."""
import numpy as np
import pytest

import tuple_fixtures as tf
from test_tuple_model import decode_entries

BOOK, D2B = tf.codebook(), tf.d2book()
FX_MAX = (1 << 53) - (1 << 29)          # rint((2 - 2^-23) * 2^52)


def keys(tb):
    return (tb[0].astype(np.uint64) << np.uint64(16)) | tb[1].astype(np.uint64)


@pytest.mark.parametrize("n", tf.SIZES)
def test_entries_are_distinct(n):
    tb = tf.dictionary(n)
    assert len(tb[0]) == n and len(np.unique(keys(tb))) == n
    assert np.all(tb[1] <= 4095)
    if n >= 16:                                   # the named entries never coincide with a bulk entry
        for name in tf.BAD:
            tb = tf.dictionary(n, {**tf.default_places(n), name: 7})
            assert len(np.unique(keys(tb))) == n, name


@pytest.mark.parametrize("n", [65537, (1 << 20) + 3, tf.TUPLES_MAX])
def test_no_power_of_two_period(n):
    """flipping any one index bit lands on an entry with another (value, counted): a decode that drops or flips a bit of
    the index cannot hit an entry of the same value"""
    fx, counted = tf.entry_fx(tf.dictionary(n), BOOK, D2B)
    i = np.arange(0, n, 1 if n < (1 << 21) else 7, dtype=np.int64)
    for k in range(n.bit_length()):
        j = i ^ (1 << k)
        m = j < n
        same = (fx[i[m]] == fx[j[m]]) & (counted[i[m]] == counted[j[m]])
        assert not same.any(), (k, i[m][same][:5])


def test_decode_is_lossless_against_decode_entries():
    n = 65537
    places = {**tf.default_places(n), **{name: 20 + k for k, name in enumerate(tf.BAD)}}
    tb = tf.dictionary(n, places)
    mine, ref = tf.decode(tb, BOOK, D2B), decode_entries(tb, BOOK, D2B)
    assert np.array_equal(np.isnan(mine), np.isnan(ref))
    assert np.array_equal(mine[~np.isnan(mine)].view(np.uint32), ref[~np.isnan(ref)].view(np.uint32))
    # every value a good entry names maps back to its code: the fp32 rows carry the whole entry
    vals = BOOK.reshape(8, 256)
    good = np.setdiff1d(np.arange(n), [places[b] for b in tf.BAD])
    for j, dim in enumerate((0, 1, 3, 4, 5, 6, 7, 8)):
        code = (tb[0][good] >> np.uint32(4 * j)) & np.uint32(15)
        col = mine[good, dim]
        assert np.array_equal(code == tf.ABSENT, np.isnan(col))
        assert np.array_equal(vals[j][code[code != tf.ABSENT]], col[code != tf.ABSENT].view(np.uint32))
    k2 = tb[1][good]
    assert np.array_equal(D2B[k2[k2 != 4095]], mine[good, 2][k2 != 4095].view(np.uint32))


def test_named_entries_decode_to_what_they_stand_for():
    n = 64
    places = {**tf.default_places(n), **{name: 20 + k for k, name in enumerate(tf.BAD)}}
    tb = tf.dictionary(n, places)
    rows = tf.decode(tb, BOOK, D2B)
    fx, counted = tf.entry_fx(tb, BOOK, D2B)
    assert (fx[places["pmax"]], fx[places["nmax"]], fx[places["pmax6"]], fx[places["nmax6"]]) == (FX_MAX, -FX_MAX, FX_MAX, -FX_MAX)
    assert all(counted[places[k]] == 1 for k in ("pmax", "nmax", "pmax6", "nmax6", "zw"))
    assert fx[places["null"]] == 0 and counted[places["null"]] == 0 and np.isnan(rows[places["null"]]).all()
    zfx, zc = tf.entry_fx(tb, BOOK, D2B, w=tf.ZERO_W)
    assert zc[places["zw"]] == 0 and zfx[places["zw"]] == 0          # only zero-weight dimensions present: null
    assert (fx[places["p2"]], fx[places["n2"]]) == (1 << 53, -(1 << 53))   # outside (-2^53, 2^53): must be refused
    # the refused entries: the empty slots decode as absent (as decode_entries reads them), the NaN value as NaN
    assert np.isnan(rows[places["d2_empty"], 2]) and np.isnan(rows[places["d2_nan"], 2])
    assert BOOK.reshape(8, 256)[tf.CODE_EMPTY] == tf.EMPTY and D2B[tf.D2_EMPTY] == tf.EMPTY
    assert np.isnan(np.uint32(BOOK.reshape(8, 256)[tf.CODE_NAN]).view(np.float32))
    assert BOOK.reshape(8, 256)[tf.CODE_NAN] != tf.EMPTY and D2B[tf.D2_NAN] != tf.EMPTY


@pytest.mark.parametrize("n", [(1 << 20) + 3, tf.TUPLES_MAX])
@pytest.mark.parametrize("T", [8192 + 8 * 5 + 3, 3 * 8192 + 77])
def test_every_group_carries_eight_high_bytes(n, T):
    C = 3
    idx = tf.hi_byte_groups(n, C, T)
    tl, th = tf.planes(idx)
    assert idx.max() < n
    assert np.array_equal(tl.astype(np.uint32) | (th.astype(np.uint32) << 16), idx)
    full = T // 8 * 8
    g = th[:, :full].reshape(C, -1, 8)
    assert all(len(set(grp)) == 8 for row in g for grp in row.tolist())            # full tiles and the ragged tail alike
    ragged = g[:, (T // tf.TILE) * tf.TILE // 8:]
    assert ragged.size and all(len(set(grp)) == 8 for row in ragged for grp in row.tolist())
    # every position of a group sees many high bytes, and the whole range is covered
    for q in range(8):
        assert len(np.unique(th[:, q:full:8])) >= min(((n - 1) >> 16) + 1, (T // 8) // 2)
    if n == tf.TUPLES_MAX and T > 2 * tf.TILE:
        assert len(np.unique(th)) == 256 and idx.max() > (1 << 23)


@pytest.mark.parametrize("n", [24574, 24575, 24576, 24577, 65537])
@pytest.mark.parametrize("T", tf.T_EDGES)
def test_boundary_indices_land_where_designed(n, T):
    C = 4
    idx = tf.boundary(n, C, T)
    special = tf.boundary_indices(n)
    assert special == {24574: [0, 24573], 24575: [0, 24574], 24576: [0, 24575], 24577: [0, 24575, 24576],
                       65537: [0, 24575, 24576, 65536]}[n]
    for c in range(C):
        for k, p in enumerate(tf.boundary_positions(T)):
            assert idx[c, p] == special[(k + c) % len(special)]
    assert idx.max() < n


def test_plane_builders_stay_in_range_and_mean_what_they_say():
    n, C, T = 65537, 3, 3 * 8192 + 100
    for name, f in tf.PLANES.items():
        idx = f(n, C, T)
        assert idx.shape == (C, T) and idx.dtype == np.uint32 and idx.max() < n, name
    w = tf.warp_uniform(n, C, T)
    blocks = w[:, :T // 256 * 256].reshape(C, -1, 256)
    for c in range(C):                                      # a whole warp on one entry: the head entry, then the last one
        for b, blk in enumerate(blocks[c]):
            if (b + c) % 3 < 2:
                assert set(blk.tolist()) == {(5, n - 1)[(b + c) % 3]}
    rf = tf.reversed_freq(n, C, T)
    assert np.mean(rf >= tf.hot(n)) > 0.99
    bp = tf.bank_pair(n, C, T)
    res = (bp[:, :T // 256 * 256].reshape(C, -1, 256) % 16)
    assert all(len(set(b.tolist())) == 1 for row in res for b in row)
    assert np.mean([len(set(b.tolist())) for row in bp[:, :T // 256 * 256].reshape(C, -1, 32) for b in row]) > 30
    for n_small in (1, 2):
        for name, f in tf.PLANES.items():
            assert f(n_small, 2, 100).max() < n_small, name


def test_max_groups_and_small_sums_by_hand():
    n, C, T = 64, 2, 80
    tb = tf.dictionary(n)
    fx, counted = tf.entry_fx(tb, BOOK, D2B)
    p = tf.default_places(n)
    idx = tf.max_groups(n, C, T)
    g = idx[0, :40].reshape(5, 8)                          # row 0: groups 0..4 are kinds 0..4
    assert list(g[0]) == [p["pmax"]] * 8 and list(g[1]) == [p["nmax"]] * 8
    assert sorted(g[2].tolist()) == sorted([p["nmax"]] * 7 + [p["null"]])
    assert sorted(g[3].tolist()) == sorted([p["nmax6"]] * 6 + [p["zw"]] + [p["null"]])
    # the sums of these groups, worked out from the per-entry values
    assert tf.expected(g[0:1], fx, counted) == ([8 * FX_MAX], [8])
    assert tf.expected(g[1:2], fx, counted) == ([-8 * FX_MAX], [8])
    assert tf.expected(g[2:3], fx, counted) == ([-7 * FX_MAX], [7])
    assert tf.expected(g[3:4], fx, counted) == ([-6 * FX_MAX + int(fx[p["zw"]])], [7])
    zfx, zc = tf.entry_fx(tb, BOOK, D2B, w=tf.ZERO_W)
    assert tf.expected(g[3:4], zfx, zc) == ([6 * int(zfx[p["nmax6"]])], [6]) and zfx[p["nmax6"]] == -FX_MAX
    # and the reference equals the oracle run on the decoded Form D tensor
    import oracle
    rows = tf.rows_of(idx, tb, BOOK, D2B)
    assert tf.expected(idx, fx, counted) == oracle.score_dims_fx(rows)
    assert tf.expected(idx, zfx, zc) == oracle.score_dims_fx(rows, w=tf.ZERO_W)


@pytest.mark.parametrize("n", [1, 2, 24577])
def test_reference_equals_the_oracle_on_the_decoded_tensor(n, orc):
    tb = tf.dictionary(n)
    for w in (None, tf.ONES_W, tf.ZERO_W):
        fx, counted = tf.entry_fx(tb, BOOK, D2B, w=w)
        for name, f in tf.PLANES.items():
            idx = f(n, 3, 8193)
            assert tf.expected(idx, fx, counted) == orc.score_dims_fx(tf.rows_of(idx, tb, BOOK, D2B), w=w), name


def test_streamed_windows_cut_the_rows():
    assert tf.stream_chunks(4096, 40_000) == 3                 # Tc = 16384: 16384 + 16384 + 7232
    assert tf.stream_chunks(3, 16385) == 1 and tf.stream_chunks(4096, 16384) == 1 and tf.stream_chunks(4096, 16385) == 2
