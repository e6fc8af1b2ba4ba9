"""CPU model of the corpus digest (tests/corpus_digest_model.py): the keys follow the oracle's dimension values, and over
oracle-generated and hand-built corpora, under default, custom and zero weights, sum count * value over the counted keys
and the per-dimension census equal the per-record sums exactly; the fixed words follow the oracle's report.  No GPU needed."""
import numpy as np
import pytest

import corpus_digest_model as dm
import corpus_fixtures as cf

W_CUSTOM = np.array([0.3, 0.1, 0.05, 0.05, 0.1, 0.1, 0.1, 0.1, 0.1])
W_ZERO = np.array([0.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])


def corpora(orc):
    gen = orc.gen_records(0x5EED0D20, orc.STREAM_CORPUS, 0, 1, 0, 6000, 300).reshape(-1)
    hand = dm.distinct_d2(1500, seed=0x5EED0D21)
    planted, _, _ = cf.planted(5000)
    return {"generated": gen, "hand": hand, "planted": planted, "saturating": cf.saturating(3000, (0, 2, 4), 2)}


@pytest.fixture(scope="module")
def cases(orc):
    return corpora(orc)


def test_keys_follow_the_oracle_dims(orc, cases):
    for name, recs in cases.items():
        d2, slots, valid = dm.keys(recs)
        for t in range(0, len(recs), 7):
            d, m = orc.reward_dims(recs[t])
            kd, km = dm.key_dims(d2[t], slots[t])
            assert km == m, (name, t)
            assert np.array_equal(np.isnan(kd), np.isnan(d)) and np.array_equal(kd[~np.isnan(kd)], d[~np.isnan(d)]), (name, t)


@pytest.mark.parametrize("w", [None, W_CUSTOM, W_ZERO], ids=["default", "custom", "zero"])
def test_counted_sums_equal_per_record_sums(orc, cases, w):
    for name, recs in cases.items():
        dig = dm.digest(recs)
        assert sum(dig.values()) == int(np.count_nonzero(recs["flags"] & 0x08))
        # per record: finalReward and the census of the counted records
        rsum = rn = 0
        dsum, dcnt = [0] * 9, [0] * 9
        for t in range(len(recs)):
            d, m, fr = orc.reward_one(recs[t], w)
            if fr is None or np.isnan(fr):
                continue
            rsum += dm.fx(fr); rn += 1
            for i in range(9):
                if not np.isnan(d[i]):
                    dsum[i] += dm.fx(d[i]); dcnt[i] += 1

        def reward(db, k):
            kd, km = dm.key_dims(db, k)
            fr = orc.final_reward(kd, km, w)
            return None if fr is None or np.isnan(fr) else dm.fx(fr)
        assert dm.weighted(dig, reward) == (rsum, rn), name
        for i in range(9):
            def dim(db, k, i=i):
                if reward(db, k) is None:
                    return None
                v = dm.key_dims(db, k)[0][i]
                return None if np.isnan(v) else dm.fx(v)
            assert dm.weighted(dig, dim) == (dsum[i], dcnt[i]), (name, i)
        ref = orc.report(recs, w=w)
        assert ref.withReward == rn and [ref.dim[i].count for i in range(9)] == dcnt


def test_fixed_words_follow_the_records(orc, cases):
    for name, recs in cases.items():
        for base in (0, (1 << 40) + 8):
            w = dm.fixed_words(orc.report(recs, idx_base=base), base)
            fb = recs["feedback"]
            assert w[:3] == [int(np.sum(fb == 1)), int(np.sum(fb == 2)), int(np.sum((fb != 1) & (fb != 2)))], name
            mode = np.where(recs["mode"] < 5, recs["mode"], 0)
            assert w[3:18] == [int(x) for m in range(5) for x in (np.sum(mode == m), np.sum((mode == m) & (fb == 1)), np.sum((mode == m) & (fb == 2)))]
            assert w[24:27] == [int(recs[f].astype(np.int64).sum()) for f in ("toolCalls", "toolSucc", "toolFail")]
            for p in range(6):
                ex = w[27 + 3 * p: 30 + 3 * p]
                nz = [x for x in ex if x != 0]
                assert nz == sorted(nz, key=lambda x: np.uint64(np.int64(x)), reverse=True) and all(x != 0 for x in ex[:len(nz)])
