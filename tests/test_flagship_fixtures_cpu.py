"""The fixtures of tests/flagship_fixtures.py reach the edges they are built for, checked without a GPU: dictionary sizes and
the count build's batches by build_twin_h's formulas, the entries at the chunk and slice edges by their counts, the nnz gate
on both sides, the wide rows' partial products past 2^64, the digest corpora's distinct VALID keys by corpus_digest_model,
and the probe keys' home slots by a Python restatement of cd_insert's hash -- itself compared with the engine's mix64,
compiled from csrc/apo_device.cuh into a host-only harness."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import corpus_digest_model as dm
import count_model as cm
import flagship_fixtures as ff
import k1_fixtures as kf

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "senweaver-ide_b200", "csrc")


def row_sets(idx, rows):
    return [set(np.unique(idx[c]).tolist()) for c in rows]


def pairs_agree(idx, rows, seed):
    """count_model.pairs summed through a random table (values and counted flags) equals the plain per-evaluation sum"""
    rank, _ = ff.rank_index(idx)
    sub = rank[list(rows)]
    rng = np.random.default_rng(seed)
    n = int(rank.max()) + 1
    tval = [cm.entry(v, f) for v, f in zip(rng.integers(-(1 << 53), 1 << 53, n), rng.integers(0, 2, n))]
    off, p = cm.pairs(sub, sub.shape[1])
    assert cm.count_sums(off, p, tval) == cm.plain_sums(sub, sub.shape[1], tval)
    return off, p


def test_cap_reaches_the_dictionary_cap_in_three_batches():
    idx = ff.cap_index()
    C, T = idx.shape
    assert (C, T) == (150, (1 << 17) + 3)
    rank, cnt = ff.rank_index(idx)
    assert len(cnt) == ff.TWIN_T_CAP and cnt.min() >= 1                          # exactly 2^20 distinct evaluations
    assert ff.batches(len(cnt), C) == (1 << 20, 64, 3, 22)
    assert ff.fixed_rank(cnt, ff.CAP_SINGLE) == ff.TWIN_T_CAP - 1 == cm.ENTRY_MAX  # the rarest: the last entry ...
    assert ff.CAP_SINGLE in set(idx[ff.CAP_SINGLE_ROW].tolist()) and ff.CAP_SINGLE_ROW >= 128   # ... in the ragged batch
    per_row = [len(np.unique(r)) for r in idx]
    assert max(per_row) <= T // 16 and ff.counts_held(sum(per_row), C, T)
    assert np.sort(cnt)[::-1][:ff.KT_HOT_MAX].sum() * 4 >= C * T * 3              # the copy's head rule
    a, b, c, d = row_sets(idx, (63, 64, 127, 128))
    assert a != b and c != d
    off, p = pairs_agree(idx, (0, 63, 64, 149), 1)
    e, n = cm.unpack(p)
    assert e.max() == cm.ENTRY_MAX and n[e == cm.ENTRY_MAX].tolist() == [1]
    over = ff.over_cap_index(idx)
    assert len(np.unique(over)) == ff.TWIN_T_CAP + 1


def test_two_batches_are_full():
    tails_n = ff.TWO_HEAD + ff.TWO_C * ff.TWO_TAIL
    _, R, nb, last = ff.batches(tails_n, ff.TWO_C)
    assert (R, nb, last) == (64, 2, 64)
    tails = [ff.TWO_HEAD + np.arange(c * ff.TWO_TAIL, (c + 1) * ff.TWO_TAIL) for c in range(ff.TWO_C)]
    idx = ff._dict_rows(0x5EEDF101, ff.TWO_C, ff.CAP_T, ff.TWO_HEAD, tails, None)
    _, cnt = ff.rank_index(idx)
    assert len(cnt) == tails_n
    per_row = [len(np.unique(r)) for r in idx]
    assert ff.counts_held(sum(per_row), ff.TWO_C, ff.CAP_T)
    assert np.sort(cnt)[::-1][:ff.KT_HOT_MAX].sum() * 4 >= idx.size * 3


def test_chunks_edges_are_known_entries():
    dims, idx, pool_of = ff.chunks()
    C, T = idx.shape
    assert T % 8 != 0
    rank, cnt = ff.rank_index(idx)
    n = len(cnt)
    assert n == 16385 and ff.batches(n, C)[0] == 16416                          # three chunks, the last holding entry 16384
    for e, k in ff.CH_EDGES.items():
        assert cnt[pool_of[e]] == k and ff.fixed_rank(cnt, pool_of[e]) == e
    for first, end, k in ff.CH_GROUPS:                                          # a group fills its index range in any order
        assert np.count_nonzero(cnt > k) == first and np.count_nonzero(cnt >= k) == end
    off, p = pairs_agree(idx, range(C), 2)
    e, _ = cm.unpack(p)
    row = [e[int(off[c]):int(off[c + 1])] for c in range(C)]
    assert (row[0] >= 2 * ff.TH_CHUNK).sum() == 1 and not ((row[0] >= ff.TH_CHUNK) & (row[0] < 2 * ff.TH_CHUNK)).any()
    assert {31, 32, 8191, 8192, 16383} <= set(row[1].tolist())
    assert ff.counts_held(len(p), C, T)
    assert len(np.unique(dims.reshape(-1, 9).view(np.uint32), axis=0)) == n       # the pool entries are distinct evaluations


@pytest.mark.parametrize("extra", [0, 1])
def test_nnz_gate_sides(extra):
    _, idx = ff.nnz_gate(extra)
    C, T = idx.shape
    nnz = sum(len(np.unique(r)) for r in idx)
    assert (C * T) % 16 == 0 and nnz == C * T // 16 + extra
    assert ff.counts_held(nnz, C, T) == (not extra)
    pairs_agree(idx, range(C), 3)


def test_wide_rows_pass_2_64(orc):
    e = ff.wide_rows()
    fx, counted = kf.fx_model(e[:, None, :])
    assert counted == [1, 1] and fx[0] == -fx[1] and abs(fx[0]) < 2 << 52      # the table's (-2, 2) range
    assert abs(fx[0]) > (2 << 52) - (1 << 31)
    d = ff.wide()
    assert d.shape == (2, ff.WIDE_T, 9)
    plus = d[:, :, 0] > 0
    assert plus.sum(axis=1).tolist() == [ff.WIDE_SPLIT[0], ff.WIDE_T]
    tval = [cm.entry(v, 1) for v in fx]
    idx = np.where(plus, 0, 1)
    off, p = cm.pairs(idx, ff.WIDE_T)
    assert off.tolist() == [0, 2, 3]
    _, n = cm.unpack(p)
    assert all(int(k) * abs(fx[0]) >= 1 << 64 for k in n)                    # every count * value past 2^64
    sums = cm.count_sums(off, p, tval)
    assert sums == [(6 * fx[0], ff.WIDE_T), (ff.WIDE_T * fx[0], ff.WIDE_T)]
    want = [sum(k * f for k, f in zip(row, fx)) for row in ff.wide_counts()]
    assert [s for s, _ in sums] == want


@pytest.mark.parametrize("T", [ff.GATE_SMALL_T, ff.GATE_LARGE_T])
def test_digest_gates(T):
    cap = ff.digest_cap(T)
    assert cap == {ff.GATE_SMALL_T: 1 << 18, ff.GATE_LARGE_T: 1 << 20}[T] and T >= ff.DIGEST_MIN
    for extra in (0, 1):
        recs = ff.gate(T, extra)
        assert len(recs) == T and len(dm.digest(recs)) == cap + extra
    if T == ff.GATE_LARGE_T:
        recs = ff.gate_invalid(T)
        d2, s, valid = dm.keys(recs)
        assert len(dm.digest(recs)) == cap
        assert len(set(zip(d2[~valid].tolist(), s[~valid].tolist()))) > cap      # far more keys on invalid records


def test_no_valid_and_few():
    recs = ff.no_valid()
    assert len(recs) >= ff.DIGEST_MIN and len(dm.digest(recs)) == 0
    for k in ff.FEW:
        recs = ff.few(k)
        assert len(recs) >= ff.DIGEST_MIN and len(dm.digest(recs)) == k


def test_probe_keys_land_where_the_model_says():
    g = ff.probe_golden()
    ns = ff.digest_slots(ff.PROBE_T)
    assert g["slots"] == ns == 1 << 21 and 0 < g["target"] < ns - 1
    recs, chain, wrap = ff.probe()
    assert len(recs) == ff.PROBE_T and len(chain) == 256 and len(wrap) == 64
    d2, s, _ = dm.keys(ff.keyed(chain + wrap, calls=ff.PROBE_CALLS, template=0))
    homes = [ff.home_slot(x, y, ns) for x, y in zip(d2.tolist(), s.tolist())]
    assert homes == [g["target"]] * 256 + [ns - 1] * 64
    dig = dm.digest(recs)
    assert all(dig[(x, y)] == 3 for x, y in zip(d2.tolist(), s.tolist()))
    assert len(dig) == 5000 + 320 <= ff.digest_cap(ff.PROBE_T)


def test_hash_constants_are_the_headers():
    """GOLD and mix64's shifts and multipliers as apo_device.cuh states them; cd_insert's home slot as apo_kernels.cu"""
    src = open(os.path.join(CSRC, "apo_device.cuh")).read()
    assert re.search(r"GOLD = 0x9E3779B97F4A7C15ull;", src)
    body = re.search(r"mix64\(unsigned long long z\) \{(.*?)return z;", src, re.S).group(1)
    assert re.findall(r"z \^= z >> (\d+);", body) == ["30", "27", "31"]
    assert re.findall(r"z \*= (0x[0-9A-F]+)ull;", body) == ["0xBF58476D1CE4E5B9", "0x94D049BB133111EB"]
    kern = open(os.path.join(CSRC, "apo_kernels.cu")).read()
    assert "uint32_t h = (uint32_t)mix64(key.x ^ mix64((unsigned long long)key.y + GOLD)) & mask;" in kern


def test_hash_model_matches_the_engines_mix64(tmp_path):
    """10^5 keys through the engine's mix64 and home slot (a host-only build of apo_device.cuh) and through the model"""
    nvcc = shutil.which("nvcc")
    if nvcc is None:
        pytest.skip("no nvcc: the constants are pinned against the header text")
    exe = str(tmp_path / "mix64_harness")
    subprocess.check_call([nvcc, "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "-I", CSRC, "-o", exe,
                           os.path.join(HERE, "c", "mix64_harness.cu")])
    rng = np.random.default_rng(0x5EEDF105)
    n, ns = 100_000, 1 << 21
    keys = rng.integers(0, 1 << 64, (n, 2), dtype=np.uint64, endpoint=False)
    keys[:1000, 1] &= np.uint64((1 << 22) - 1)                                  # slots as the digest packs them
    keys[1000:2000, 0] = (rng.uniform(-1, 1, 1000)).view(np.uint64)             # d2 bit patterns
    keys[2000:2004] = [[0, 0], [2 ** 64 - 1, 2 ** 64 - 1], [1, 0], [0, 1]]
    inp = np.array([n, ns], np.uint64).tobytes() + keys.tobytes()
    out = np.frombuffer(subprocess.run([exe], input=inp, capture_output=True, check=True).stdout, np.uint64).reshape(n, 2)
    for (x, y), (mx, h) in zip(keys.tolist(), out.tolist()):
        assert ff.mix64(x) == mx and ff.home_slot(x, y, ns) == h
