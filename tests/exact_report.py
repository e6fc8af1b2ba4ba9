"""The exact corpus report (apo_corpus_report) of Form R records, and a bit-for-bit comparison with it.

oracle.report sums finalReward and the nine dimensions in sequential binary64, as the reference does, so its sums and
averages drift from the exact ones by up to ~n * 2^-53 * sum|v|, and a dimension whose average sits on a flag threshold
(-0.5, -0.3, 0) can land on either side of it.  The engine sums rint(v * 2^52) exactly and rounds each sum once.  The exact
report takes:

- every count, rate, pattern, example and tool total from oracle.report (integers, and rates of integers rounded once);
- withReward, rewardSum, avgReward and every dim[i] field from the exact fixed-point integers of oracle/candidates.py
  (cand_records / cand_generated(records=True)), rounded once (fx_to_double) with the report rules of dimstat;
- every pattern's severity from its rule (APO:650,676,700,720,741,761): the engine writes it for every pattern; oracle.report
  leaves it 0 when no record is 'bad' (the APO:641 early out), where no pattern is emitted.

The two oracles count the same records: exact_report asserts that their shared integers agree.

check_exact(rep, want) compares every field of a report struct (the engine's CorpusReport, or oracle.Report) with the exact
report: integers equal, binary64 fields by their bytes (NaN included).  No tolerance, no threshold waiver.

Plain helpers, imported by the tests that use them (no fixtures, no GPU)."""
import struct

import numpy as np

import oracle
from oracle import candidates

NDIM, NPAT, NMODE = oracle.NDIM, oracle.NPAT, oracle.NMODE
DIM_FLAGS = ("low_flag", "low_severity", "sugg_flag", "sugg_priority")
MINC = (2, 2, 3, 2, 2, 2)                                  # APO:645,671,695,715,736,756
BIG = 1 << 20                                              # from here on oracle.report runs on a thread pool (same integers)


def pattern_severity(p, count):
    """APO:650,676,700,720,741,761"""
    if p in (0, 1):
        return 2 if count >= 5 else 1
    if p == 3:
        return 2
    if p == 4:
        return 2 if count >= 4 else 1
    return 1


def combine(ref, fx):
    """the exact report from oracle.report's struct `ref` and the exact breakdown `fx` (a dict of oracle/candidates.py) of
    the same records"""
    shared = ("total", "good", "bad", "none", "withReward")
    assert tuple(int(getattr(ref, f)) for f in shared) == tuple(fx[f] for f in shared), "the oracles counted different records"
    assert [int(ref.dim[i].count) for i in range(NDIM)] == [fx["dim"][i]["count"] for i in range(NDIM)]
    pats = []
    for p in range(NPAT):
        n = int(ref.pat[p].count)
        pats.append({"count": n, "flag": int(n >= MINC[p]), "severity": pattern_severity(p, n),
                     "examples": [int(x) for x in ref.pat[p].examples]})
        assert int(ref.pat[p].flag) == pats[-1]["flag"]
        assert int(ref.bad) == 0 or int(ref.pat[p].severity) == pats[-1]["severity"]
    return {"total": fx["total"], "good": fx["good"], "bad": fx["bad"], "none": fx["none"], "goodRate": ref.goodRate,
            "byMode": [[int(x) for x in ref.byMode[m]] for m in range(NMODE)],
            "byModeGoodRate": [ref.byModeGoodRate[m] for m in range(NMODE)],
            "withReward": fx["withReward"], "rewardFx": fx["rewardFx"], "rewardSum": fx["rewardSum"], "avgReward": fx["avgReward"],
            "dim": [{k: fx["dim"][i][k] for k in ("fx", "sum", "count", "avg") + DIM_FLAGS} for i in range(NDIM)],
            "pat": pats,
            "toolCalls": int(ref.toolCalls), "toolSucc": int(ref.toolSucc), "toolFail": int(ref.toolFail),
            "toolSuccessRate": ref.toolSuccessRate}


def exact_report(recs, idx_base=0, w=None):
    """the exact corpus report of Form R records `recs` (examples numbered from idx_base), under weights w (default: the
    reference's)"""
    recs = np.ascontiguousarray(recs, oracle.RECORD_DTYPE).reshape(-1)
    ref = oracle.report(recs, idx_base=idx_base, w=w, nthreads=16 if len(recs) >= BIG else 0)
    return combine(ref, candidates.cand_records(recs[None], idx_base=idx_base, w=w)[0])


def exact_rows(rows, idx_base=0, w=None):
    """one exact report per row of Form R records [C][T] (the per-candidate corpus reports)"""
    return [exact_report(r, idx_base, w) for r in rows]


def exact_generated(seed, cands, T, agent_permille=300, w=None, nthreads=16):
    """the exact corpus reports of the generated rollout rows `cands` over [0, T) (apo_rollouts_generate /
    apo_rollouts16_generate): exact sums from cand_generated(records=True), the rest from oracle.report of each row"""
    fx = candidates.cand_generated(seed, cands, 0, T, agent_permille, w=w, nthreads=nthreads, records=True)
    out = []
    for c, d in zip(cands, fx):
        row = oracle.gen_records(seed, oracle.STREAM_ROLLOUT, int(c), 1, 0, T, agent_permille, nthreads).reshape(-1)
        out.append(combine(oracle.report(row, w=w, nthreads=nthreads), d))
        del row
    return out


def _bits(x):
    return struct.pack("<d", float(x))


def _hex(x):
    return f"{float(x)!r} ({_bits(x)[::-1].hex()})"


def diff_exact(rep, want):
    """[(field, got, want)] for every field of the report struct `rep` that differs from the exact report `want`: integers by
    value, binary64 fields by their bytes"""
    out = []

    def num(name, got, exp):
        if int(got) != int(exp):
            out.append((name, int(got), int(exp)))

    def f64(name, got, exp):
        if _bits(got) != _bits(exp):
            out.append((name, float(got), float(exp)))

    for f in ("total", "good", "bad", "none", "withReward", "toolCalls", "toolSucc", "toolFail"):
        num(f, getattr(rep, f), want[f])
    for f in ("goodRate", "rewardSum", "avgReward", "toolSuccessRate"):
        f64(f, getattr(rep, f), want[f])
    for m in range(NMODE):
        for k in range(3):
            num(f"byMode[{m}][{k}]", rep.byMode[m][k], want["byMode"][m][k])
        f64(f"byModeGoodRate[{m}]", rep.byModeGoodRate[m], want["byModeGoodRate"][m])
    for i in range(NDIM):
        a, b = rep.dim[i], want["dim"][i]
        f64(f"dim[{i}].sum", a.sum, b["sum"])
        f64(f"dim[{i}].avg", a.avg, b["avg"])
        for f in ("count",) + DIM_FLAGS:
            num(f"dim[{i}].{f}", getattr(a, f), b[f])
    for p in range(NPAT):
        a, b = rep.pat[p], want["pat"][p]
        for f in ("count", "flag", "severity"):
            num(f"pat[{p}].{f}", getattr(a, f), b[f])
        for k in range(3):
            num(f"pat[{p}].examples[{k}]", a.examples[k], b["examples"][k])
    return out


def check_exact(rep, want, what=""):
    d = diff_exact(rep, want)
    assert not d, f"{what}: " + "; ".join(f"{n}: got {_hex(g) if isinstance(g, float) else g}, "
                                          f"want {_hex(e) if isinstance(e, float) else e}" for n, g, e in d[:12])


# ------------------------------------------------------------------------------------------------ threshold fixtures
F_ERRORS, F_ENDED, F_VALID = 0x01, 0x02, 0x08


def record(**kw):
    """one VALID 'good' chat-mode record (mode 1: the non-agent thresholds) where every dimension is present at 1.0, with the
    fields of kw changed"""
    r = np.zeros(1, oracle.RECORD_DTYPE)
    base = dict(feedback=1, flags=F_VALID | F_ENDED, mode=1, userMsgs=1, asstMsgs=1, toolCalls=1, toolSucc=1, toolFail=0,
                llmCalls=1, tokens=500, toolDurMs=100.0)
    base.update(kw)
    for k, v in base.items():
        r[k] = v
    return r


def _rows(*parts):
    return np.concatenate([np.repeat(record(**kw), n) for n, kw in parts])


BAD_TOOLS = dict(feedback=2, toolCalls=4)


def threshold_fixtures():
    """[(name, records, dim, edge, side, flags)]: corpora of a few records that put dimension `dim`'s exact average on
    `side` ("at", "below" or "above") of the flag threshold `edge`; flags = that dimension's (low_flag, low_severity,
    sugg_flag, sugg_priority) the exact average calls for.  Level values (oracle/apo_oracle.c orc_reward_dims, mode 1):
    d3 -0.5 at 2 failed tool calls, -1 at 3; d4 -0.3 at 7..10 calls; d6 1 - 0.4 * (llmCalls - 1), clamped at -1; d7 0 at
    5001..10000 tokens, -0.5 above 10000; d8 -0.3 at 5..6 turns."""
    return [
        # d3 at exactly -0.5, the low_severity / sugg_priority boundary: flagged, severity 1 (needs < -0.5)
        ("d3_at_-0.5", _rows((6, dict(BAD_TOOLS, toolSucc=2, toolFail=2))), 3, -0.5, "at", (1, 1, 1, 1)),
        # ... and one record at -1 more: below -0.5, severity 2
        ("d3_below_-0.5", _rows((6, dict(BAD_TOOLS, toolSucc=2, toolFail=2)), (1, dict(BAD_TOOLS, toolSucc=1, toolFail=3))),
         3, -0.5, "below", (1, 2, 1, 2)),
        # rint(-0.3 * 2^52) = -0.3 * 2^52 - 0.25: five (six) records at -0.3 average to the double below -0.3 (flagged),
        # where the sequential binary64 sum gives -0.3 itself
        ("d4_-0.3_x5", _rows((5, dict(toolCalls=8, toolSucc=8))), 4, -0.3, "below", (1, 1, 1, 1)),
        ("d8_-0.3_x5", _rows((5, dict(userMsgs=5, asstMsgs=5))), 8, -0.3, "below", (1, 1, 1, 1)),
        ("d8_-0.3_x6", _rows((6, dict(userMsgs=6, asstMsgs=6))), 8, -0.3, "below", (1, 1, 1, 1)),
        # exactly 0.0: not flagged (sugg_flag needs < 0)
        ("d7_at_0", _rows((4, dict(tokens=6000))), 7, 0.0, "at", (0, 1, 0, 1)),
        ("d0_at_0", _rows((3, dict()), (3, dict(feedback=2))), 0, 0.0, "at", (0, 1, 0, 1)),
        # d6 levels: 0.6 and -0.6000000000000001 cancel exactly in fixed point (sequential binary64: -1.1e-16, flagged)
        ("d6_0.6_-0.6", _rows((2, dict(llmCalls=2)), (2, dict(llmCalls=5))), 6, 0.0, "at", (0, 1, 0, 1)),
        # 0.19999999999999996 and -0.20000000000000018: one unit of 2^-52 below 0
        ("d6_0.2_-0.2", _rows((2, dict(llmCalls=3)), (2, dict(llmCalls=4))), 6, 0.0, "below", (0, 1, 1, 1)),
        ("d6_every_level", _rows(*[(1, dict(llmCalls=k)) for k in range(1, 8)]), 6, 0.0, "below", (0, 1, 1, 1)),
        # counts around low_flag's count >= 5 (d3 at -1) and sugg_flag's count >= 3 (d7 at -0.5)
        ("d3_-1_x4", _rows((4, dict(BAD_TOOLS, toolSucc=1, toolFail=3))), 3, -0.3, "below", (0, 2, 1, 2)),
        ("d3_-1_x5", _rows((5, dict(BAD_TOOLS, toolSucc=1, toolFail=3))), 3, -0.3, "below", (1, 2, 1, 2)),
        ("d7_-0.5_x2", _rows((2, dict(tokens=20_000))), 7, 0.0, "below", (0, 1, 0, 1)),
        ("d7_-0.5_x3", _rows((3, dict(tokens=20_000))), 7, 0.0, "below", (0, 1, 1, 1)),
    ]


def padded(recs, T):
    """recs followed by T - len(recs) records that carry no reward ('none' feedback, VALID clear): every dimension's sums
    and counts stay those of recs"""
    pad = np.repeat(record(feedback=0, flags=0), T - len(recs))
    return np.concatenate([recs, pad])


DYADIC_W = np.array([0.25, 0.125, 0.125, 0.125, 0.125, 0.0625, 0.0625, 0.0625, 0.0625])     # sums to 1


def dyadic(T, seed=0):
    """T VALID records whose every dimension is present at a level that is a multiple of 1/2 (d1 never 0.8, d2 -1 / 1 from
    two tool calls, d3 never -0.2, d4, d6 and d8 at 1), so that under DYADIC_W every finalReward is a multiple of 1/32 and
    every term and partial sum of the report is exact in binary64"""
    rng = np.random.default_rng(seed)
    r = np.repeat(record(), T)
    r["feedback"] = rng.integers(0, 3, T)
    r["flags"] = F_VALID | np.where(rng.random(T) < 0.5, F_ERRORS, 0)               # never 'ended without errors' (d1 0.8)
    r["mode"] = rng.integers(0, 2, T) * 3                                              # modes 0 and 3: the chat thresholds
    r["toolCalls"] = 2                                                                 # d4 1 (needs <= 3)
    r["toolFail"] = rng.choice([0, 2], T)                                              # d2 1 / -1, d3 1 / -0.5
    r["toolSucc"] = 2 - r["toolFail"]
    r["toolDurMs"] = 2 * rng.choice([100.0, 2000.0, 5000.0, 20000.0], T)               # d5 1, 0.5, 0, -0.5
    r["tokens"] = rng.choice([500, 3000, 8000, 20000], T)                              # d7 1, 0.5, 0, -0.5
    return r
