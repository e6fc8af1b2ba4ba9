"""The model of the paired comparison per record group (tests/group_pair_fixtures.py) on the CPU: every fixture reaches its
edge, the model's sums are the exact rational ones, summed over the labels it is pair_fixtures' model and at G = 1 it is
that model field for field; and the beam service's rules: vsReferenceByGroup, evaluateBeam(groupPairs=True) and
runBeamSearch(withGroupComparison=True), with their ValueErrors; and the TypeScript decoder's offsets against the C struct,
with the option on the addon and the service contract."""
import importlib

import numpy as np
import pytest

import group_pair_fixtures as gf
import pair_fixtures as pf
from extremes_fixtures import final_rewards

FIX = {f[0]: f for f in gf.all_fixtures()}


@pytest.mark.parametrize("name", sorted(FIX))
def test_summed_over_groups_is_the_pair_model(name):
    _, dims, refs, w, lab, G = FIX[name]
    fr, ok = final_rewards(dims, w)
    m = gf.group_pair_model(fr, ok, refs, lab, G)
    whole = pf.pair_model(fr, ok, refs)
    for c, row in enumerate(m):
        assert len(row) == G
        assert gf.summed(row) == {f: int(whole[c][f]) for f in gf.INT_FIELDS}, c
        assert all(x["ref"] == whole[c]["ref"] for x in row)
    one = gf.group_pair_model(fr, ok, refs, np.zeros(dims.shape[1], np.uint8), 1)
    assert [r[0] for r in one] == whole or all(                      # field for field, NaN included
        repr(sorted(a.items())) == repr(sorted(b.items())) for a, b in zip([r[0] for r in one], whole))


@pytest.mark.parametrize("name", ["shapes_mod5", "one_unit_lanes", "rn_edges_runs", "extreme_alt", "nulls_1025_tail1"])
def test_model_sums_agree_with_fractions(name):
    _, dims, refs, w, lab, G = FIX[name]
    fr, ok = final_rewards(dims, w)
    m = gf.group_pair_model(fr, ok, refs, lab, G)
    for c, r in enumerate(int(v) for v in refs):
        if r == gf.NONE:
            continue
        for g in range(min(G, 6)):
            sel = lab[: dims.shape[1]] == g
            assert pf.fraction_sums(fr, ok & sel[None, :], c, r) == (m[c][g]["D1"], m[c][g]["D2"]), (c, g)


def test_fixtures_reach_their_edges():
    _, dims, refs, w, lab, G = FIX["extreme_alt"]
    fr, ok = final_rewards(dims, w)
    m = gf.group_pair_model(fr, ok, refs, lab, G)
    assert m[0][0]["D1"] > 0 and m[1][0]["D1"] < 0                 # a pair and its mirror in each label
    assert m[0][0]["D1"] == -m[1][0]["D1"] and m[0][1]["D2"] == m[1][1]["D2"]
    big = gf.group_pair_model(*final_rewards(pf.extreme(), w), refs, (np.arange((1 << 22) + 3) % 2).astype(np.uint8), 2)
    assert big[0][0]["D1"] > 2 ** 83 and big[0][0]["D2"] > 2 ** 128 and big[0][1]["D1"] > 2 ** 83
    lab64, G64 = gf.labels("lanes", 1024)
    assert G64 == 64 and len(set(lab64[:32].tolist())) == 32        # every lane its own label
    labe, Ge = gf.labels("ends", 4096)
    assert set(labe.tolist()) == {0, Ge - 1}
    for r in pf.TAILS:                                               # a label holding only each row's last evaluations
        T = 1024 + r
        name = f"nulls_{T}_tail{r or 1}"
        _, dims, refs, w, lab, G = FIX[name]
        assert lab[T - 1] == 1 and lab[: T - max(r, 1)].max() == 0
        m = gf.group_pair_model(*final_rewards(dims, w), refs, lab, G)
        # row 0's last evaluation is null: in label 1 the pair (0, 1) has refOnly = 1 when only that position is held
        if r <= 1:
            assert m[0][1]["refOnly"] == 1 and m[0][1]["n"] == 0
    shp = FIX["shapes_mod5"]
    m = gf.group_pair_model(*final_rewards(shp[1], shp[3]), shp[2], shp[4], shp[5])
    assert all(x["ref"] == gf.NONE and x["n"] == 0 for x in m[0])   # PAIR_NONE in every group
    assert all(x["ties"] == x["n"] and x["D1"] == 0 for x in m[7])  # a self-pair in every group


class _FakeEngine:
    """Returns a scripted ScoreResult with pairs and per-group pairs when asked for them"""

    def __init__(self, eng):
        self.eng, self.calls, self.refs, self.G = eng, [], [], 0

    def dims_upload(self, dims):
        self.C = dims.shape[0]

    def record_groups_upload(self, labels, G=0):
        self.G = G

    def candidate_refs_upload(self, refs):
        self.refs.append([int(r) for r in refs])

    def score(self, C, K, source=0, candidates=False, groups=False, pairs=False, group_pairs=False):
        self.calls.append((candidates, groups, pairs, group_pairs))
        m = self.eng
        scores = np.array([0.1 * c for c in range(C)])
        topk = np.argsort(-scores, kind="stable")[:K].astype(np.int32)
        cands = (m.CandidateReport * C)() if candidates else None
        refs = self.refs[-1] if self.refs else [m.PAIR_NONE] * C
        prs = (m.CandidatePair * C)() if pairs else None
        gps = ((m.CandidatePair * max(self.G, 1)) * C)() if group_pairs else None
        for c in range(C):
            for x in ([prs[c]] if pairs else []) + (list(gps[c]) if group_pairs else []):
                x.ref = refs[c]
                x.meanDiff = x.variance = x.stdDev = x.stdErr = float("nan")
        if group_pairs:
            for c in range(C):
                if refs[c] != m.PAIR_NONE:
                    gps[c][0].n, gps[c][0].wins, gps[c][0].meanDiff = 1, 1, 0.25
                    gps[c][1].n, gps[c][1].losses, gps[c][1].ties = 3, 2, 1
                    gps[c][1].meanDiff, gps[c][1].stdErr = -0.5, 0.125
        return m.ScoreResult(scores, np.full(C, 10, np.uint64), topk, None, None, cands, groups=None, pairs=prs, group_pairs=gps)


def _svc():
    svc_mod = importlib.import_module("senweaver-ide_b200.apo_service")
    eng = importlib.import_module("senweaver-ide_b200.engine")
    fake = _FakeEngine(eng)
    return svc_mod, eng, fake, svc_mod.APOService(fake, None)


def test_vs_reference_by_group():
    _, eng, fake, svc = _svc()
    N = eng.PAIR_NONE
    refs = [N, 0, 0, 1]
    cands = [{"version": f"v{c}", "content": str(c)} for c in range(4)]
    res = svc.evaluateBeam(cands, dims=np.zeros((4, 6, 9), np.float32), reports=True, groups=(np.zeros(6), ["heldOut", "seen"]),
                           refs=refs, groupPairs=True)
    assert fake.calls == [(True, True, True, True)]
    assert svc.candidateReport(res, 0)["vsReferenceByGroup"] is None
    by = svc.candidateReport(res, 3)["vsReferenceByGroup"]
    assert set(by) == {"heldOut", "seen"}
    assert by["heldOut"] == {"reference": 1, "pairedRollouts": 1, "wins": 1, "losses": 0, "ties": 0, "meanRewardDiff": 0.25, "diffStdErr": None}
    assert by["seen"] == {"reference": 1, "pairedRollouts": 3, "wins": 0, "losses": 2, "ties": 1, "meanRewardDiff": -0.5, "diffStdErr": 0.125}
    assert svc.getBeamState()["beam"][0]["version"] == "v3"          # adoption still by the means alone
    for bad in ({"refs": refs}, {"groups": (np.zeros(6), ["a"])}, {}):
        with pytest.raises(ValueError):
            svc.evaluateBeam(cands, dims=np.zeros((4, 6, 9), np.float32), reports=True, groupPairs=True, **bad)
    plain = svc.evaluateBeam(cands, dims=np.zeros((4, 6, 9), np.float32), reports=True, refs=refs)
    assert "vsReferenceByGroup" not in svc.candidateReport(plain, 1)


def test_beam_search_with_group_comparison():
    _, eng, fake, svc = _svc()
    seen = []

    def propose(parent, n, report=None):
        seen.append(report)
        return [parent["content"] + f"/{k}" for k in range(n)]

    dims = lambda cands: np.zeros((len(cands), 6, 9), np.float32)         # noqa: E731
    groups = (np.array([0, 0, 0, 1, 1, 1]), ["seen", "heldOut"])
    svc.runBeamSearch("seed", propose, dims, rounds=2, withReports=True, rolloutGroups=groups, withParentComparison=True,
                      withGroupComparison=True)
    assert fake.calls and all(c == (True, True, True, True) for c in fake.calls)
    assert any(r is not None and "vsReferenceByGroup" in r for r in seen)
    fake.calls.clear()
    svc.runBeamSearch("seed", propose, dims, rounds=1, withReports=True, rolloutGroups=groups, withParentComparison=True)
    assert fake.calls == [(True, True, True, False)]                  # default: no per-group comparison
    for kw in ({"withReports": True, "withParentComparison": True}, {"withReports": True, "rolloutGroups": groups},
               {"rolloutGroups": groups, "withParentComparison": True}):
        with pytest.raises(ValueError):
            svc.runBeamSearch("seed", propose, dims, rounds=1, withGroupComparison=True, **kw)


def test_ts_decoder_and_addon_surface():
    """decodeCandidateGroupPairs reads the 128-byte pair record at (c * G + g) * 128 with the offsets the C struct has (the same
    pinned constants as decodeCandidatePairs); the service contract, renderer proxy, main-process service and addon carry the
    candidateGroupPairs option and block, and the proxy adds it to the channel arguments only when asked for"""
    import ctypes
    import os
    eng = importlib.import_module("senweaver-ide_b200.engine")
    P = eng.CandidatePair
    assert ctypes.sizeof(P) == 128 and eng.SCORE_CANDIDATE_GROUP_PAIRS == 0x200 and "apo_candidate_group_pairs" in eng.ABI_SYMBOLS
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = open(os.path.join(root, "ts", "candidateReportCodec.ts")).read()
    pins = {"CANDIDATE_PAIR_BYTES": ctypes.sizeof(P), "OFF_PR_REF": P.ref.offset, "OFF_PR_N": P.n.offset, "OFF_PR_WINS": P.wins.offset,
            "OFF_PR_LOSSES": P.losses.offset, "OFF_PR_TIES": P.ties.offset, "OFF_PR_CAND_ONLY": P.candOnly.offset,
            "OFF_PR_REF_ONLY": P.refOnly.offset, "OFF_PR_SUM_LO": P.sumLo.offset, "OFF_PR_SUM_HI": P.sumHi.offset,
            "OFF_PR_SUM_SQ": P.sumSq.offset, "OFF_PR_MEAN_DIFF": P.meanDiff.offset, "OFF_PR_VARIANCE": P.variance.offset,
            "OFF_PR_STD_DEV": P.stdDev.offset, "OFF_PR_STD_ERR": P.stdErr.offset}
    for name, value in pins.items():
        assert f"const {name} = {value};" in src, (name, value)
    assert "export function decodeCandidateGroupPairs(buf: VSBuffer, C: number, G: number): CandidatePair[][]" in src
    assert "decodePair(buf, (c * G + g) * CANDIDATE_PAIR_BYTES, c)" in src        # [C][G], row-major as the C output
    assert "decodePair(buf, c * CANDIDATE_PAIR_BYTES, c)" in src
    svc = open(os.path.join(root, "ts", "apoScoringService.ts")).read()
    assert "candidateGroupPairs?: VSBuffer;" in svc and "candidateGroupPairs?: number;" in svc
    assert svc.count("candidateGroupPairs?: number): Promise<ApoScoreBlocks>;") == 3
    assert svc.count("if (candidateGroupPairs) {") == 3                        # only then a longer argument list
    main = open(os.path.join(root, "ts", "apoScoringMainService.ts")).read()
    assert "candidateGroupPairs?: ArrayBuffer" in main and main.count("candidateGroupPairs ?? 0));") == 3
    assert "out.candidateGroupPairs = VSBuffer.wrap" in main
    napi = open(os.path.join(root, "napi", "apo_napi.c")).read()
    assert '"candidateGroupPairs"' in napi and napi.count("APO_SCORE_CANDIDATE_GROUP_PAIRS") >= 3
    jobs = open(os.path.join(root, "napi", "apo_jobs.h")).read()
    assert "#define APO_JOB_CANDIDATE_GROUP_PAIRS_MAX_BYTES (1ull << 32)" in jobs
