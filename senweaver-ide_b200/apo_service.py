"""Host-side mirror of the reference's APOService API (APO:203-267).

Same method names, argument meaning and error behaviour as
src/vs/workbench/contrib/senweaver/common/apoService.ts; the reductions run on the GPU
engine through the C ABI:

    _buildReport / _analyzePatterns (APO:498-625, 635-773) -> Engine.score(corpus=True)   (k_detect6)
    beam evaluation + top-K (server side in the reference, consumed at APO:1138-1166)
                                                         -> Engine.score                 (k_reward9 + radix top-K)

Everything that is text or CRUD (descriptions, suggestions, segments, config) stays on the
host, as in the reference.  Async reference methods are plain methods here; failures are
swallowed with a `[APO]` warning and an empty result, never raised (APO:1211-1214).
"""
from __future__ import annotations

import copy
import json
import math
import time
import uuid

import numpy as np

from .engine import DIM_NAMES, GROUPS_MAX, MODE_NAMES, PAIR_NONE, SRC_DIMS, SRC_ROLLOUTS, Engine
from .jsfmt import js_substring, js_to_fixed
from .trace_collector import TraceCollectorService

APO_STORAGE_KEY, APO_CONFIG_KEY, APO_SEGMENTS_KEY = "senweaver.apo.data", "senweaver.apo.config", "senweaver.apo.segments"
APO_BEAM_KEY, APO_GRADIENTS_KEY = "senweaver.apo.beamState", "senweaver.apo.gradients"   # APO:360,364
MAX_REPORTS, MAX_SUGGESTIONS, MAX_GRADIENTS = 50, 200, 50                # APO:276-277, 405
DEFAULT_APO_CONFIG = {                                                   # APO:279-292
    "enabled": True, "autoAnalyzeEnabled": True, "autoAnalyzeIntervalMs": 3600000, "minTracesForAnalysis": 20,
    "minFeedbacksForAnalysis": 10, "autoApplySuggestions": False, "uploadOptimizationsToServer": True,
    "beamWidth": 4, "branchFactor": 4, "beamRounds": 3, "gradientBatchSize": 4,
}
SEVERITY = ("low", "medium", "high")
DIM_CATEGORY = {                                                         # APO:576-586
    "tool_success_rate": "tool_usage", "tool_call_reliability": "tool_usage", "tool_call_efficiency": "tool_usage",
    "tool_duration_efficiency": "tool_usage", "token_efficiency": "context_management",
    "response_efficiency": "core_behavior", "conversation_efficiency": "core_behavior",
    "task_completion": "core_behavior", "user_feedback": "core_behavior",
}
PATTERN_TEXT = (                                                          # order of APO:643-770
    ("Negative feedback follows conversations in which errors occurred", "core_behavior"),
    ("Failed tool calls precede user dissatisfaction", "tool_usage"),
    ("High token consumption coincides with poor feedback", "context_management"),
    ("Several LLM calls (likely retries) still end in dissatisfaction", "core_behavior"),
    ("Long multi-turn conversations still end in dissatisfaction", "core_behavior"),
    ("Slow tool execution (>15 s total) coincides with dissatisfaction", "tool_usage"),
)


def _first_preview(trace, type_):
    for sp in trace["spans"]:
        if sp["type"] == type_:
            return sp["data"].get("contentPreview") or ""
    return ""


def _js_constant(name):
    return {"Infinity": math.inf, "-Infinity": -math.inf, "NaN": math.nan}[name]


def _finite_or_none(obj):
    """What JSON.stringify does to non-finite numbers (they become null), applied recursively."""
    if isinstance(obj, float) and not math.isfinite(obj):
        return None
    if isinstance(obj, dict):
        return {k: _finite_or_none(v) for k, v in obj.items()}
    if isinstance(obj, list):
        return [_finite_or_none(v) for v in obj]
    return obj


class APOService:
    def __init__(self, engine: Engine, traceCollectorService: TraceCollectorService, storageService=None,
                 productService=None, requestService=None):
        self._engine, self._tc = engine, traceCollectorService
        self._storage, self._product, self._request = storageService, productService, requestService
        self._reports, self._suggestions, self._segments = [], [], []
        self._config = dict(DEFAULT_APO_CONFIG)
        self._beamState, self._textualGradients = None, []
        self._stateListeners, self._suggestionListeners = [], []
        self._dirty = False
        self._lastRolloutCount = 0
        self._groupNames = None                                               # names of the record groups of the last evaluateBeam
        api = (getattr(productService, "senweaverApiConfig", None) or {}).get("apiBaseUrl") if productService else None
        self._apoApiUrl = f"{api or 'https://ide-api.senweaver.com'}/api/apo"          # APO:328-329
        self._loadFromStorage()

    # ---- events
    def onDidChangeState(self, fn):
        self._stateListeners.append(fn)

    def onDidGenerateSuggestions(self, fn):
        self._suggestionListeners.append(fn)

    def _fire(self, listeners, *a):
        for fn in list(listeners):
            try:
                fn(*a)
            except Exception:
                pass

    # ---- analysis (APO:477-496)
    def analyzePromptEffectiveness(self):
        report = self._buildReport(self._tc.getAllTraces())
        self._reports.append(report)
        self._dirty = True
        self._saveToStorage()
        if self._config["uploadOptimizationsToServer"] and self._request is not None:
            try:                                                               # APO:1345-1356, silent on failure
                self._request(f"{self._apoApiUrl}/report", {"version": "1.0.0", "report": report})
            except Exception:
                pass
        self._fire(self._stateListeners)
        return report

    def _corpus_report(self, traces):
        """Two corpus passes when some trace changed after it was scored (reward statistics use the
        snapshot the reward was computed from, tallies and patterns the live counters); one otherwise."""
        eng = self._engine
        eng.dims_upload(np.full((1, 4, 9), np.nan, np.float32))
        live = self._tc.corpus_records(traces)
        eng.corpus_upload(live)
        rep = eng.score(1, 0, corpus=True).report
        snap = self._tc.corpus_records(traces, scored=True)
        if snap.tobytes() != live.tobytes():
            eng.corpus_upload(snap)
            rew = eng.score(1, 0, corpus=True).report
        else:
            rew = rep
        return rep, rew

    def _buildReport(self, traces):
        now = time.time() * 1000.0
        starts = [t["startTime"] for t in traces]
        if traces:
            rep, rew = self._corpus_report(traces)
            good, bad, none = int(rep.good), int(rep.bad), int(rep.none)
            goodRate = float(rep.goodRate)
            byMode = self._byMode(rep)
            avgReward = None if rew.withReward == 0 else float(rew.avgReward)
            rewardByDimension = self._rewardByDimension(rew)
        else:
            rep = rew = None
            good = bad = none = 0
            goodRate, byMode, avgReward, rewardByDimension = 0, {}, None, {}

        patterns = []
        if rep is not None:
            def example(p, gi):
                t = traces[gi]
                return {"threadId": t["threadId"], "userMessagePreview": _first_preview(t, "user_message"),
                        "assistantMessagePreview": self._example_detail(p, t), "feedback": t["summary"]["userFeedback"]}
            patterns = self._emittedPatterns(rep, example)
            patterns.extend(self._dimensionPatterns(rew))

        suggestions = self._generateLocalSuggestions(goodRate, patterns, byMode, avgReward, rew)
        report = {"id": str(uuid.uuid4()), "generatedAt": now,
                  "period": {"from": min(starts) if starts else now, "to": (max(starts) if starts else 0) or now},
                  "totalConversations": len(traces), "goodFeedbackCount": good, "badFeedbackCount": bad,
                  "noFeedbackCount": none, "goodRate": goodRate, "byMode": byMode, "patterns": patterns,
                  "suggestions": suggestions, "avgReward": avgReward, "rewardByDimension": rewardByDimension}
        self._suggestions.extend(suggestions)
        self._suggestions = self._suggestions[-MAX_SUGGESTIONS:]
        if suggestions:
            self._fire(self._suggestionListeners, suggestions)
        return report

    @staticmethod
    def _byMode(rep):
        """APO:519-544: per-mode tallies of a corpus report, modes without records left out."""
        byMode = {}
        for m, name in enumerate(MODE_NAMES):
            tot, g, b = (int(x) for x in rep.byMode[m])
            if tot:
                byMode[name] = {"total": tot, "good": g, "bad": b, "goodRate": float(rep.byModeGoodRate[m])}
        return byMode

    @staticmethod
    def _emittedPatterns(rep, example):
        """APO:643-770: the emitted problem patterns of a corpus report; example(p, index) shapes one of its first three
        matching records."""
        patterns = []
        for p in range(6):
            q = rep.pat[p]
            if not q.flag:
                continue
            text, cat = PATTERN_TEXT[p]
            ex = [example(p, int(gi)) for gi in q.examples if gi >= 0]
            patterns.append({"id": str(uuid.uuid4()), "description": text, "frequency": int(q.count),
                             "severity": SEVERITY[q.severity], "relatedCategory": cat, "examples": ex})
        return patterns

    @staticmethod
    def _rewardByDimension(rew):
        """APO:556-568 from a corpus report or a candidate report (same apo_dimstat fields)."""
        return {DIM_NAMES[i]: {"sum": float(rew.dim[i].sum), "count": int(rew.dim[i].count), "avg": float(rew.dim[i].avg)}
                for i in range(9) if rew.dim[i].count}

    @staticmethod
    def _dimensionPatterns(rew):
        """APO:574-596: the dimension-low patterns of a corpus report or a candidate report."""
        out = []
        for i, name in enumerate(DIM_NAMES):
            d = rew.dim[i]
            if d.count and d.low_flag:
                out.append({"id": str(uuid.uuid4()),
                            "description": f"{name} dimension reward signal consistently low (avg: {js_to_fixed(d.avg, 3)})",
                            "frequency": int(d.count), "severity": SEVERITY[d.low_severity],
                            "relatedCategory": DIM_CATEGORY.get(name, "core_behavior"), "examples": []})
        return out

    def candidateReport(self, res, c, groupNames=None):
        """The report of one beam candidate, shaped like _buildReport's, from a ScoreResult scored with the per-candidate
        breakdown (evaluateBeam(..., reports=True)): feedback tallies and goodRate of its rollouts, avgReward (== its score),
        rewardByDimension, the dimension-low patterns and the suggestions they raise (the rules of APO:574-596, 800-827, by
        the code _buildReport uses), and badExamples = the first three rollout indices with 'bad' feedback.
        When the result also carries the candidate's corpus report (rollout records scored with candidate_corpus=True,
        evaluateBeam(..., patterns=True)), the report adds byMode, the six problem patterns of APO:643-770 (examples = rollout
        indices) ahead of the dimension-low ones, and toolStats (TCS:603-624); its suggestions then follow the pattern and
        mode rules of APO:830-859 as well.  When the result carries the per-candidate extremes (extremes=True), the report
        adds lowestRollouts / highestRollouts: the candidate's 32 lowest- and highest-reward rollouts as {"index", "finalReward"}
        (reward ascending / descending, ties -> lower index), the sample runs the critique step reads; the caller looks the
        rollouts up by index.  When the result carries the per-candidate group scores (evaluateBeam(..., groups=(labels, names))),
        the report adds byGroup: {name: {totalRollouts, goodFeedbackCount, badFeedbackCount, goodRate, avgReward}} over the
        candidate's rollouts in each record group (avgReward None when none of them has a reward); names default to those of the
        last evaluateBeam.  When the result carries the per-candidate reward spread (evaluateBeam(..., spread=True)), the report
        adds rewardStdDev (the sample standard deviation of its rollouts' rewards) and scoreStdErr (the standard error of
        avgReward), both None with fewer than two rewarded rollouts: the scale against which a gap between two candidates'
        scores can be read.  Pure: it neither records the suggestions nor fires events nor touches storage."""
        cc = res.candidate_corpus[c] if getattr(res, "candidate_corpus", None) is not None else None
        r = res.candidates[c] if res.candidates is not None else cc
        goodRate = float(r.goodRate)
        avgReward = None if r.withReward == 0 else float(r.avgReward)
        byMode = self._byMode(cc) if cc is not None else {}
        patterns = self._emittedPatterns(cc, lambda p, gi: gi) if cc is not None else []
        patterns.extend(self._dimensionPatterns(r))
        out = {"candidate": int(c), "totalRollouts": int(r.total), "goodFeedbackCount": int(r.good), "badFeedbackCount": int(r.bad),
               "noFeedbackCount": int(r.none), "goodRate": goodRate, "avgReward": avgReward,
               "rewardByDimension": self._rewardByDimension(r), "patterns": patterns,
               "suggestions": self._generateLocalSuggestions(goodRate, patterns, byMode, avgReward, r)}
        if res.candidates is not None:
            out["badExamples"] = [int(x) for x in r.badExamples if x >= 0]
        if cc is not None:
            out["byMode"] = byMode
            out["toolStats"] = {"totalToolCalls": int(cc.toolCalls), "totalToolSucceeded": int(cc.toolSucc),
                                "totalToolFailed": int(cc.toolFail),
                                "toolSuccessRate": None if cc.toolCalls == 0 else float(cc.toolSuccessRate)}
        ex = res.extremes[c] if getattr(res, "extremes", None) is not None else None
        if ex is not None:
            n = int(ex.n)
            out["lowestRollouts"] = [{"index": int(ex.lowest[i]), "finalReward": float(ex.lowestReward[i])} for i in range(n)]
            out["highestRollouts"] = [{"index": int(ex.highest[i]), "finalReward": float(ex.highestReward[i])} for i in range(n)]
        gs = res.groups[c] if getattr(res, "groups", None) is not None else None
        if gs is not None:
            names = groupNames if groupNames is not None else (self._groupNames or [str(g) for g in range(len(gs))])
            out["byGroup"] = {names[g]: {"totalRollouts": int(x.total), "goodFeedbackCount": int(x.good), "badFeedbackCount": int(x.bad),
                                         "goodRate": float(x.goodRate), "avgReward": None if x.withReward == 0 else float(x.avgReward)}
                              for g, x in enumerate(gs)}
        sp = res.spread[c] if getattr(res, "spread", None) is not None else None
        if sp is not None:
            out["rewardStdDev"] = None if sp.n < 2 else float(sp.stdDev)
            out["scoreStdErr"] = None if sp.n < 2 else float(sp.stdErr)
        pr = res.pairs[c] if getattr(res, "pairs", None) is not None else None
        if pr is not None:
            out["vsReference"] = None if pr.ref == PAIR_NONE else self._vsReference(pr)
        gp = res.group_pairs[c] if getattr(res, "group_pairs", None) is not None else None
        if gp is not None:
            names = groupNames if groupNames is not None else (self._groupNames or [str(g) for g in range(len(gp))])
            out["vsReferenceByGroup"] = None if gp[0].ref == PAIR_NONE else {names[g]: self._vsReference(x) for g, x in enumerate(gp)}
        return out

    @staticmethod
    def _vsReference(pr):
        """the vsReference dict of one apo_candidate_pair (whole record axis or one group)"""
        return {"reference": int(pr.ref), "pairedRollouts": int(pr.n), "wins": int(pr.wins), "losses": int(pr.losses), "ties": int(pr.ties),
                "meanRewardDiff": None if pr.n == 0 else float(pr.meanDiff), "diffStdErr": None if pr.n < 2 else float(pr.stdErr)}

    @staticmethod
    def parentRefs(cands, carried):
        """refs of a round's candidates for the paired comparison: each child (cands[carried:]) names its parent's index in
        cands; the beam members carried over (cands[:carried], the seed among them) name none."""
        index = {x["version"]: i for i, x in enumerate(cands)}
        return np.array([PAIR_NONE if i < carried else index.get(x.get("parentVersion"), PAIR_NONE) for i, x in enumerate(cands)],
                        np.uint32)

    @staticmethod
    def _checkGroups(groups):
        """(labels, names) of evaluateBeam / runBeamSearch: one uint8 label per rollout index, names unique, 1..GROUPS_MAX of them."""
        labels, names = groups
        names = list(names)
        if not 1 <= len(names) <= GROUPS_MAX or len(set(names)) != len(names):
            raise ValueError(f"record groups need 1..{GROUPS_MAX} unique names, got {names!r}")
        return np.ascontiguousarray(labels, np.uint8).reshape(-1), names

    @staticmethod
    def _example_detail(p, t):
        s = t["summary"]
        if p == 0:
            return _first_preview(t, "assistant_message")
        if p == 1:
            for sp in t["spans"]:
                if sp["type"] == "tool_call" and sp["data"].get("toolSuccess") is False:
                    return f"Tool {sp['data'].get('toolName')} failed: {(sp['data'].get('toolResult') or '')[:100]}"
            return "Tool undefined failed: "
        if p == 2:
            return f"Total tokens: {s['totalTokens']}"
        if p == 3:
            return f"LLM calls: {s['totalLLMCalls']}"
        if p == 4:
            return f"Conversation turns: {sum(1 for sp in t['spans'] if sp['type'] == 'user_message')}"
        return f"Tool duration: {js_to_fixed(s['totalToolDurationMs'] / 1000, 1)}s"

    def _generateLocalSuggestions(self, goodRate, patterns, byMode, avgReward, rew):
        """APO:775-862: thresholds from the engine's flags, text on the host."""
        out = []

        def add(cat, prio, desc, why, impact):
            out.append({"id": str(uuid.uuid4()), "targetCategory": cat, "type": "modify", "priority": prio,
                        "description": desc, "reasoning": why, "estimatedImpact": impact, "status": "pending"})

        if 0 < goodRate < 0.5:                                               # APO:785
            extra = f" (avg reward: {js_to_fixed(avgReward, 3)})" if avgReward is not None else ""
            add("core_behavior", "high", f"Overall approval rate is only {js_to_fixed(goodRate * 100, 1)}%{extra}; the prompt needs a broad revision",
                "An approval rate under 50% points at a systemic prompt problem", "approval rate +10-20%")
        if rew is not None:
            for i, name in enumerate(DIM_NAMES):                             # APO:800-827
                d = rew.dim[i]
                if d.count and d.sugg_flag:
                    add(DIM_CATEGORY.get(name, "core_behavior"), SEVERITY[d.sugg_priority],
                        f"{name} dimension performing poorly (avg: {js_to_fixed(d.avg, 3)}, n={d.count})",
                        f"The {name} reward dimension is negative on average", f"{name} reward +0.2-0.5")
        for p in patterns:                                                   # APO:830-843
            if p["severity"] == "high":
                add(p["relatedCategory"], "high", f"High-frequency issue: {p['description']} (occurred {p['frequency']} times)",
                    "Frequent, severe pattern: tighten the related prompt rules", f"about {min(p['frequency'], 5)} fewer such cases")
        for mode, st in byMode.items():                                      # APO:846-859
            if st["total"] >= 5 and st["goodRate"] < 0.3:
                o = {"id": str(uuid.uuid4()), "targetCategory": "mode_specific", "type": "modify", "priority": "medium",
                     "description": f"{mode} mode approval rate is only {js_to_fixed(st['goodRate'] * 100, 1)}%",
                     "reasoning": "This mode is well below the average approval rate", "estimatedImpact": f"better {mode} mode approval",
                     "status": "pending"}
                out.append(o)
        return out

    # ---- beam evaluation: the step the reference delegates to its backend --------------------------------
    def evaluateBeam(self, candidates, dims=None, rollouts=None, reports=False, patterns=False, extremes=False, groups=None,
                     spread=False, refs=None, groupPairs=False):
        """Score a beam of VersionedPromptTemplate candidates on their rollout outcomes and keep the
        top `beamWidth` (score desc, ties -> lower index), then apply the APO:1138-1166 update with the
        strict `>` adoption rule (APO:1159).  dims: float32 [C][T][9] (NaN = absent) or rollouts:
        apo_record [C][T].  reports=True also builds the per-candidate breakdown (res.candidates, see
        candidateReport); with rollouts, reports=True and patterns=True also build every candidate's corpus
        report (res.candidate_corpus: problem patterns, per-mode tallies, tool totals).  extremes=True also lists every
        candidate's 32 lowest- and highest-reward rollouts (res.extremes).  groups=(labels, names) also splits every candidate's
        rollouts by record group (res.groups [C][G]): labels[t] < len(names) is the group of rollout index t.  spread=True also
        builds every candidate's reward spread (res.spread: exact sums, variance, standard deviation and standard error).
        refs (uint32 [C], a candidate index or PAIR_NONE each) also compares every candidate with its reference on the rollouts
        both were scored on (res.pairs: wins, losses, ties, the exact paired sums, meanDiff and its standard error).
        groupPairs=True (which needs groups and refs) also makes that comparison per record group (res.group_pairs [C][G]).  The
        adoption rule stays the strict `>` on the means."""
        if groupPairs and (groups is None or refs is None):
            raise ValueError("evaluateBeam: groupPairs needs groups and refs (the comparison is split by the groups' labels)")
        try:
            C = len(candidates)
            K = min(self._config["beamWidth"], C)
            extra = {"candidates": True} if reports else {}
            if reports and patterns and rollouts is not None:
                extra["candidate_corpus"] = True
            if extremes:
                extra["extremes"] = True
            if groups is not None:
                labels, names = self._checkGroups(groups)
                self._engine.record_groups_upload(labels, len(names))
                self._groupNames = names
                extra["groups"] = True
            if spread:
                extra["spread"] = True
            if refs is not None:
                self._engine.candidate_refs_upload(refs)
                extra["pairs"] = True
            if groupPairs:
                extra["group_pairs"] = True
            if dims is not None:
                self._engine.dims_upload(np.ascontiguousarray(dims, np.float32))
                res = self._engine.score(C, K, source=SRC_DIMS, **extra)
            else:
                self._engine.rollouts_upload(rollouts)
                res = self._engine.score(C, K, source=SRC_ROLLOUTS, **extra)
            beam = []
            for c in res.topk:
                tpl = dict(candidates[int(c)])
                tpl["score"] = None if math.isinf(res.scores[c]) else float(res.scores[c])
                beam.append(tpl)
            best = beam[0] if beam and beam[0]["score"] is not None else None
            self._applyBeamUpdate({"beam": beam, "bestPrompt": best, "bestScore": best["score"] if best else None,
                                   "round": (self._beamState["currentRound"] + 1) if self._beamState else 1})
            return res
        except Exception as e:
            print("[APO] Beam evaluation failed:", e)
            return None

    def runBeamSearch(self, seedPrompt, proposeCandidates, rolloutDims=None, rounds=None, withReports=False, rolloutRecords=None,
                      withExtremes=False, rolloutGroups=None, withSpread=False, withParentComparison=False, withGroupComparison=False):
        """Client-side round driver (SURVEY 8f rank 3) around the GPU top-K: each round expands every beam
        member into `branchFactor` children through the caller's `proposeCandidates(parent, n) -> [content]`
        hook (the LLM critique/edit step of APO:918-988 lives there), scores parents + children on
        `rolloutDims(candidates) -> float32 [C][T][9]` or `rolloutRecords(candidates) -> apo_record [C][T]` (exactly
        one of the two), keeps the top `beamWidth` and applies the APO:1138-1166 update.  withReports=True calls
        `proposeCandidates(parent, n, report)` instead, with the candidateReport of the parent from the round that
        scored it (None for the unscored seed), so that the critique can name what the parent lost on; with
        rolloutRecords that report also carries the parent's problem patterns, byMode and toolStats; withExtremes=True
        (which needs withReports=True) adds the parent's lowestRollouts / highestRollouts, indices into the rollouts the
        caller scored it on; rolloutGroups=(labels, names) (which needs withReports=True too) adds the parent's byGroup, so that
        a label that marks a held-out part of the rollouts shows whether a child improved only where its critique looked;
        withSpread=True (which needs withReports=True too) adds the parent's rewardStdDev / scoreStdErr, so that the critique
        can tell a lead from the noise of the rollouts; withParentComparison=True (which needs withReports=True too) adds the
        parent's vsReference: how it fared against its own parent on the rollouts that scored both (wins, losses, ties, the
        mean reward difference and its paired standard error); withGroupComparison=True (which needs withReports=True,
        rolloutGroups and withParentComparison=True) adds the parent's vsReferenceByGroup: that comparison on each group's
        rollouts, so that the critique sees whether the parent beat its own parent on the held-out ones by more than the paired
        noise there.  Returns the final beam state."""
        if (rolloutDims is None) == (rolloutRecords is None):
            raise ValueError("runBeamSearch needs exactly one of rolloutDims / rolloutRecords")
        if withExtremes and not withReports:
            raise ValueError("runBeamSearch: withExtremes needs withReports=True (the lists travel in the candidate reports)")
        if withSpread and not withReports:
            raise ValueError("runBeamSearch: withSpread needs withReports=True (the spreads travel in the candidate reports)")
        if withParentComparison and not withReports:
            raise ValueError("runBeamSearch: withParentComparison needs withReports=True (the comparisons travel in the candidate reports)")
        if rolloutGroups is not None:
            if not withReports:
                raise ValueError("runBeamSearch: rolloutGroups needs withReports=True (the group scores travel in the candidate reports)")
            rolloutGroups = self._checkGroups(rolloutGroups)
        if withGroupComparison and not (withReports and rolloutGroups is not None and withParentComparison):
            raise ValueError("runBeamSearch: withGroupComparison needs withReports=True, rolloutGroups and withParentComparison=True")
        rounds = rounds or self._config["beamRounds"]
        beam = [{"version": "v0", "content": seedPrompt, "score": None, "createdAt": time.time() * 1000.0}]
        counter = 0
        reports = {}                                                         # version -> candidateReport of its last scoring
        for _ in range(rounds):
            cands = list(beam)
            for parent in beam:
                proposed = (proposeCandidates(parent, self._config["branchFactor"], reports.get(parent["version"])) if withReports
                            else proposeCandidates(parent, self._config["branchFactor"]))
                for content in proposed:
                    counter += 1
                    cands.append({"version": f"v{counter}", "content": content, "score": None,
                                  "parentVersion": parent["version"], "createdAt": time.time() * 1000.0})
            refs = self.parentRefs(cands, len(beam)) if withParentComparison else None
            if rolloutRecords is not None:
                res = self.evaluateBeam(cands, rollouts=rolloutRecords(cands), reports=withReports, patterns=withReports,
                                        extremes=withExtremes, groups=rolloutGroups, spread=withSpread, refs=refs,
                                        groupPairs=withGroupComparison)
            else:
                res = self.evaluateBeam(cands, dims=rolloutDims(cands), reports=withReports, extremes=withExtremes, groups=rolloutGroups,
                                        spread=withSpread, refs=refs, groupPairs=withGroupComparison)
            if res is None:
                break
            if withReports:
                reports = {cands[int(c)]["version"]: self.candidateReport(res, int(c)) for c in res.topk}
            beam = self._beamState["beam"]
            self._beamState["versionCounter"] = counter
        return self.getBeamState()

    def _applyBeamUpdate(self, bu, notify=True):
        now = time.time() * 1000.0
        if self._beamState is None:                                          # APO:1141-1152
            self._beamState = {"currentRound": 0, "totalRounds": self._config["beamRounds"], "beam": [],
                               "historyBestPrompt": None, "historyBestScore": -math.inf, "versionCounter": 0,
                               "startedAt": now, "lastUpdatedAt": now}
        st = self._beamState
        if bu.get("beam"):
            st["beam"] = bu["beam"]
        if bu.get("round") is not None:
            st["currentRound"] = bu["round"]
        # a beam state reloaded before its first score carries null here (JSON.stringify(-Infinity)); `x > null` compares with 0 in JS
        incumbent = 0 if st["historyBestScore"] is None else st["historyBestScore"]
        if bu.get("bestPrompt") and bu.get("bestScore") is not None and bu["bestScore"] > incumbent:                # strict, APO:1159
            st["historyBestPrompt"], st["historyBestScore"] = bu["bestPrompt"], bu["bestScore"]
            self._applyBeamBestPrompt(bu["bestPrompt"])
        st["lastUpdatedAt"] = now
        self._dirty = True
        if notify:
            self._saveToStorage()
            self._fire(self._stateListeners)

    def _applyBeamBestPrompt(self, best):
        """APO:1219-1264: '- ' lines become individual optimized segments; otherwise replace/add one."""
        now = time.time() * 1000.0
        rules = [ln for ln in best["content"].split("\n") if ln.strip().startswith("- ")]

        def new_seg(content):
            return {"id": str(uuid.uuid4()), "category": "core_behavior", "content": content, "isActive": True,
                    "isOptimized": True, "version": 1, "createdAt": now, "updatedAt": now}

        if not rules:
            seg = next((s for s in self._segments if s["category"] == "core_behavior" and s["isActive"]), None)
            if seg:
                seg["originalContent"] = seg.get("originalContent") or seg["content"]
                seg.update(content=best["content"], isOptimized=True, version=seg["version"] + 1, updatedAt=now)
            else:
                self._segments.append(new_seg(best["content"]))
            return
        for r in rules:
            text = r.strip()[1:].strip()
            if text and not any(s["isActive"] and s["content"] == text for s in self._segments):
                self._segments.append(new_seg(text))

    def requestOptimizationFromServer(self):
        """APO:992-1215: POST {apo}/optimize with the v2.0.0 payload; the reply's suggestions join the local list as
        pending, its beamUpdate goes through the strict-greater adoption rule, its textualGradient is stored (and its
        editedPrompt becomes one more pending suggestion).  Any failure: warn and return [] (APO:1211-1214)."""
        try:
            if not self._reports:
                self.analyzePromptEffectiveness()
            if not self._reports:
                return []
            payload = self.buildOptimizePayload()
            if self._request is None:
                raise RuntimeError("no request service")
            reply = self._request(f"{self._apoApiUrl}/optimize", payload)
            if not isinstance(reply, dict):
                reply = {}
            if (reply.get("statusCode") or 0) >= 400:
                print("[APO] Server optimization request failed:", reply["statusCode"])
                return []
            sugg = list(reply.get("suggestions") or [])
            for s in sugg:
                s["id"] = s.get("id") or str(uuid.uuid4())
                s["status"] = "pending"
                self._suggestions.append(s)
            if reply.get("beamUpdate"):
                self._applyBeamUpdate(reply["beamUpdate"], notify=False)
            tgr = reply.get("textualGradient") or {}
            if tgr.get("critique"):
                best = (self._beamState or {}).get("historyBestPrompt") or {}
                tg = {"id": str(uuid.uuid4()), "promptVersion": best.get("version") or "v0", "critique": tgr["critique"],
                      "rolloutSummary": f"Based on {self._lastRolloutCount} rollouts",
                      "createdAt": time.time() * 1000.0}
                self._textualGradients.append(tg)
                self._textualGradients = self._textualGradients[-MAX_GRADIENTS:]
                if tgr.get("editedPrompt"):
                    edit = {"id": str(uuid.uuid4()), "targetCategory": "core_behavior", "type": "modify", "priority": "high",
                            "description": f"Textual Gradient optimization: {js_substring(tg['critique'], 0, 100)}...",
                            "suggestedContent": tgr["editedPrompt"], "reasoning": tg["critique"],
                            "estimatedImpact": "Prompt optimization based on Textual Gradient", "status": "pending",
                            "promptVersion": tg["promptVersion"]}
                    sugg.append(edit)
                    self._suggestions.append(edit)
            self._dirty = True
            self._saveToStorage()
            if sugg:
                self._fire(self._suggestionListeners, sugg)
            self._fire(self._stateListeners)
            return sugg
        except Exception as e:
            print("[APO] Server optimization request failed:", e)
            return []

    def requestTextualGradient(self):
        """APO:1268-1343: POST {apo}/gradient with both prompts and the gradientBatchSize most recent rated rollouts;
        the reply's critique becomes a TextualGradient, its editedPrompt (if any) a pending high-priority suggestion."""
        try:
            recent = sorted([t for t in self._tc.getAllTraces() if t["summary"]["userFeedback"] is not None],
                            key=lambda t: -t["startTime"])[: self._config["gradientBatchSize"]]
            if len(recent) < 2:
                return None
            rollouts = self._convertTracesToRolloutResults(recent)
            rules = self.getOptimizedRules()
            payload = {"version": "2.0.0", "action": "textual_gradient",
                       "textualGradientPrompt": self._buildTextualGradientPrompt(rules, rollouts),
                       "applyEditPrompt": self._buildApplyEditPrompt(rules, "{{critique_placeholder}}"),
                       "rolloutResults": rollouts, "currentRules": rules}
            if self._request is None:
                raise RuntimeError("no request service")
            reply = self._request(f"{self._apoApiUrl}/gradient", payload)
            if not isinstance(reply, dict) or (reply.get("statusCode") or 0) >= 400 or not reply.get("critique"):
                return None
            acc = 0
            for r in rollouts:
                acc = acc + (r["finalReward"] or 0)
            best = (self._beamState or {}).get("historyBestPrompt") or {}
            tg = {"id": str(uuid.uuid4()), "promptVersion": best.get("version") or "v0", "critique": reply["critique"],
                  "rolloutSummary": f"Based on {len(rollouts)} rollouts, avg reward: {js_to_fixed(acc / len(rollouts), 3)}",
                  "createdAt": time.time() * 1000.0}
            self._textualGradients.append(tg)
            if reply.get("editedPrompt"):
                sug = {"id": str(uuid.uuid4()), "targetCategory": "core_behavior", "type": "modify", "priority": "high",
                       "description": f"Textual Gradient: {js_substring(tg['critique'], 0, 100)}...", "suggestedContent": reply["editedPrompt"],
                       "reasoning": tg["critique"], "estimatedImpact": "Prompt optimization based on Textual Gradient",
                       "status": "pending", "promptVersion": tg["promptVersion"]}
                self._suggestions.append(sug)
                self._fire(self._suggestionListeners, [sug])
            self._touched()
            return tg
        except Exception as e:
            print("[APO] Textual gradient request failed:", e)
            return None

    # ---- candidate-generation hooks (SURVEY 8f rank 3): the two prompts of the textual-gradient loop ----------
    NO_RULES = "(No optimized prompt rules currently active)"

    @staticmethod
    def _experiment_block(i, r):
        """One '--- Experiment i ---' block, field for field and digit for digit as APO:926-941
        (toFixed(3) reward, toFixed(0) percent and milliseconds, toFixed(2) dims, 200-unit message previews)."""
        status = {"succeeded": "\u2705 Succeeded", "failed": "\u274c Failed"}.get(r["status"], "\u2753 Unknown")
        reward = "N/A" if r["finalReward"] is None else js_to_fixed(r["finalReward"], 3)
        msgs = "\n    ".join(f"[{m['role']}] {js_substring(m['content'], 0, 200)}" for m in r["messages"])
        tc = r["toolCallStats"]
        if tc["totalCalls"] > 0:
            rate = "N/A" if tc["successRate"] is None else js_to_fixed(tc["successRate"] * 100, 0) + "%"
            tool = (f"Tool Calls: {tc['totalCalls']} ({tc['succeeded']} succeeded, {tc['failed']} failed, rate: {rate}, "
                    f"duration: {js_to_fixed(tc['totalDurationMs'], 0)}ms)")
        else:
            tool = "Tool Calls: none"
        dims = ("Reward Dims: " + ", ".join(f"{d['name']}={js_to_fixed(d['value'], 2)}" for d in r["rewardDimensions"])) if r["rewardDimensions"] else ""
        llm = f"LLM Calls: {r['llmStats']['totalCalls']}, Tokens: {r['llmStats']['totalTokens']}"
        return (f"--- Experiment {i + 1} ---\nStatus: {status}\nFinal Reward: {reward}\nChat Mode: {r['chatMode']}\n{tool}\n{llm}\n{dims}\n"
                f"Messages:\n    {msgs}")

    def _buildTextualGradientPrompt(self, currentPromptRules, rolloutResults):
        """APO:918-962 ("textual gradient": critique the current rules from sample runs).  The section layout and
        the experiment blocks follow the reference; the instruction prose is this build's own wording."""
        rules = "\n".join(currentPromptRules) if currentPromptRules else self.NO_RULES
        experiments = "\n\n".join(self._experiment_block(i, r) for i, r in enumerate(rolloutResults))
        return ("You are an expert prompt engineer improving the system prompt of a coding-IDE assistant.\n\n"
                f"## Current Prompt Rules\n{rules}\n\n## Sample Runs with Current Prompt\n{experiments}\n\n"
                "## Your Task\nWrite a short critique: name the specific causes of the failures above and what would raise the reward "
                "next time.\nAnswer with a bullet list of concrete, testable changes (format, constraints, ordering, definitions), looking at:\n"
                "1. Structure: missing goals, contradictions, absent stop conditions\n"
                "2. Instruction quality: vague verbs, no hierarchy, overlapping scope\n"
                "3. Control and behaviour: tool limits, handling of uncertainty, verbosity\n"
                "4. Input/output specification: missing defaults, inconsistent formats\n"
                "5. Scope and safety: scope creep, unsafe actions, error handling\n\n"
                "Be direct. Fewer than 350 words.")

    def _buildApplyEditPrompt(self, currentPromptRules, critique):
        """APO:966-988 ("apply edit": rewrite the rules under the critique); reply format `- rule` per line, which is
        what _applyBeamBestPrompt splits on (APO:1226-1229)."""
        rules = "\n".join(currentPromptRules) if currentPromptRules else self.NO_RULES
        return ("Revise the prompt rules below, treating the critique as both constraint and guide.\n\n"
                "## Revision Rules\n"
                "1. Rewrite or restructure the prompt where the critique calls for it.\n"
                "2. State any requested output format, structure or word limit explicitly.\n"
                "3. Put the mechanism first: what to do, then how.\n"
                "4. Stay close to the original in tone, length and structure.\n"
                "5. Concentrate on the single most important issue raised.\n\n"
                f"## Current Prompt Rules\n{rules}\n\n## Critique\n{critique}\n\n"
                "Return only the improved prompt rules, without explanations or headers.\n"
                'Each rule goes on its own line and starts with "- ".')

    # ---- wire formats after the path (SURVEY 8f rank 2) ---------------------------------------------------
    def _convertTracesToRolloutResults(self, traces):
        """APO:866-914: trace -> RolloutResultForAPO (field for field)."""
        out = []
        for t in traces:
            msgs = []
            for sp in t["spans"]:
                d = sp["data"]
                if sp["type"] == "user_message":
                    msgs.append({"role": "user", "content": d.get("contentPreview") or ""})
                elif sp["type"] == "assistant_message":
                    msgs.append({"role": "assistant", "content": d.get("contentPreview") or ""})
                elif sp["type"] == "tool_call":
                    msgs.append({"role": "tool", "content": d.get("toolResult") or "", "toolName": d.get("toolName"),
                                 "toolSuccess": d.get("toolSuccess")})
            sm = t["summary"]
            fb = sm["userFeedback"]
            status = "succeeded" if fb == "good" else ("failed" if fb == "bad" or sm["hasErrors"] else "unknown")
            total = sm["toolCallsSucceeded"] + sm["toolCallsFailed"]
            md = t.get("metadata") or {}
            out.append({"traceId": t["id"], "threadId": t["threadId"], "status": status, "finalReward": sm["finalReward"],
                        "rewardDimensions": sm.get("rewardDimensions") or [], "messages": msgs,
                        "chatMode": md.get("chatMode") or "unknown",
                        "toolCallStats": {"totalCalls": total, "succeeded": sm["toolCallsSucceeded"], "failed": sm["toolCallsFailed"],
                                          "successRate": sm["toolCallsSucceeded"] / total if total > 0 else None,
                                          "byToolName": sm["toolCallsByName"], "totalDurationMs": sm["totalToolDurationMs"]},
                        "llmStats": {"totalCalls": sm["totalLLMCalls"], "totalTokens": sm["totalTokens"]}})
        return out

    def buildOptimizePayload(self):
        """The v2.0.0 /api/apo/optimize payload of APO:1011-1100; its rewardSummary / toolCallSummary
        reductions (APO:1051-1099) run on the engine over the same recent-feedback selection
        (feedback != null, startTime desc, first gradientBatchSize*4; APO:1003-1007)."""
        report = self.getLatestReport() or self.analyzePromptEffectiveness()
        recent = sorted([t for t in self._tc.getAllTraces() if t["summary"]["userFeedback"] is not None],
                        key=lambda t: -t["startTime"])[: self._config["gradientBatchSize"] * 4]
        rollouts = self._convertTracesToRolloutResults(recent)
        self._lastRolloutCount = len(rollouts)                                 # rolloutResults.length before the slice(0, 20)
        reward_summary = {"totalWithReward": 0, "avgFinalReward": None, "rewardDimensionAvg": {}}
        tool_summary = {"totalCalls": 0, "totalSucceeded": 0, "totalFailed": 0, "successRate": None, "totalDurationMs": 0, "byToolName": {}}
        if recent:
            self._engine.dims_upload(np.full((1, 4, 9), np.nan, np.float32))
            self._engine.corpus_upload(self._tc.corpus_records(recent, scored=True))
            rep = self._engine.score(1, 0, corpus=True).report
            reward_summary = {"totalWithReward": int(rep.withReward),
                              "avgFinalReward": None if rep.withReward == 0 else float(rep.avgReward),
                              "rewardDimensionAvg": {DIM_NAMES[i]: float(rep.dim[i].avg) for i in range(9) if rep.dim[i].count}}
            by = {}
            for r in rollouts:
                for name, st in r["toolCallStats"]["byToolName"].items():
                    e = by.setdefault(name, {"total": 0, "succeeded": 0, "failed": 0})
                    for k in e:
                        e[k] += st[k]
            self._engine.corpus_upload(self._tc.corpus_records(recent))           # tool totals read the live counters (APO:1081-1084)
            live = self._engine.score(1, 0, corpus=True).report
            succ, fail = int(live.toolSucc), int(live.toolFail)
            tool_summary = {"totalCalls": succ + fail, "totalSucceeded": succ, "totalFailed": fail,
                            "successRate": succ / (succ + fail) if succ + fail > 0 else None,
                            "totalDurationMs": sum(r["toolCallStats"]["totalDurationMs"] for r in rollouts), "byToolName": by}
        st = self._beamState
        return {"version": "2.0.0",
                "report": {k: report[k] for k in ("id", "generatedAt", "totalConversations", "goodRate", "goodFeedbackCount",
                                                  "badFeedbackCount", "byMode", "patterns")},
                "rolloutResults": rollouts[:20],
                "currentSegments": [{"id": s["id"], "category": s["category"], "content": s["content"][:1000],
                                     "isOptimized": s["isOptimized"], "version": s["version"]} for s in self.getActiveSegments()],
                "textualGradientPrompt": self._buildTextualGradientPrompt(self.getOptimizedRules(), rollouts[: self._config["gradientBatchSize"]]),
                "beamConfig": {k: self._config[k] for k in ("beamWidth", "branchFactor", "beamRounds")},
                "beamState": None if st is None else {"currentRound": st["currentRound"], "historyBestScore": st["historyBestScore"],
                                                      "beamSize": len(st["beam"])},
                "badExamples": [e for p in report["patterns"] for e in p["examples"]][:10],
                "rewardSummary": reward_summary, "toolCallSummary": tool_summary}

    # ---- segments / suggestions (APO:1360-1458)
    def getActiveSegments(self):
        return [s for s in self._segments if s["isActive"]]

    def getOptimizedPromptForCategory(self, category):
        seg = next((s for s in self._segments if s["isActive"] and s["isOptimized"] and s["category"] == category), None)
        return (seg["content"] or None) if seg else None                       # first match only (APO:1364-1367)

    def getOptimizedRules(self):
        return [s["content"] for s in self._segments if s["isActive"] and s["isOptimized"]]

    def _find(self, sid):
        return next((s for s in self._suggestions if s["id"] == sid), None)

    def _touched(self):
        self._dirty = True
        self._saveToStorage()
        self._fire(self._stateListeners)

    def applySuggestion(self, suggestionId):
        """APO:1375-1411: 'modify' rewrites the targeted (or first active same-category) segment and keeps the
        original for revert; 'add' appends a new optimized segment; anything else only changes status."""
        s = self._find(suggestionId)
        if not s or s["status"] != "pending":
            return
        now = time.time() * 1000.0
        s["status"], s["appliedAt"] = "applied", now
        if s.get("suggestedContent"):
            if s.get("targetSegmentId"):
                seg = next((g for g in self._segments if g["id"] == s["targetSegmentId"]), None)
            else:
                seg = next((g for g in self._segments if g["category"] == s["targetCategory"] and g["isActive"]), None)
            if seg is not None and s.get("type") == "modify":
                seg["originalContent"] = seg.get("originalContent") or seg["content"]
                seg["content"], seg["isOptimized"] = s["suggestedContent"], True
                seg["version"] += 1
                seg["updatedAt"] = now
            elif s.get("type") == "add":
                self._segments.append({"id": str(uuid.uuid4()), "category": s["targetCategory"], "content": s["suggestedContent"],
                                       "isActive": True, "isOptimized": True, "version": 1, "createdAt": now, "updatedAt": now})
        self._touched()

    def rejectSuggestion(self, suggestionId):
        s = self._find(suggestionId)
        if not s or s["status"] != "pending":
            return
        s["status"] = "rejected"
        self._touched()

    def revertSuggestion(self, suggestionId):
        """APO:1423-1458: restore the segment's original content (by id, else by category for 'modify'), or remove the
        segment an 'add' created (matched by category + content)."""
        s = self._find(suggestionId)
        if not s or s["status"] != "applied":
            return

        def restore(seg):
            if seg is not None and seg.get("originalContent"):
                seg["content"] = seg["originalContent"]
                seg.pop("originalContent", None)
                seg["isOptimized"] = False
                seg["version"] += 1
                seg["updatedAt"] = time.time() * 1000.0
        if s.get("targetSegmentId"):
            restore(next((g for g in self._segments if g["id"] == s["targetSegmentId"]), None))
        elif s.get("type") == "modify":
            restore(next((g for g in self._segments if g["category"] == s["targetCategory"] and g["isActive"] and g["isOptimized"]), None))
        elif s.get("type") == "add":
            self._segments = [g for g in self._segments
                              if not (g["category"] == s["targetCategory"] and g["isOptimized"] and g["content"] == s.get("suggestedContent"))]
        s["status"] = "reverted"
        self._touched()

    # ---- rule injection (SURVEY 8f rank 4): the consumer of getOptimizedRules in the system-prompt builder
    def packOptimizedRules(self, maxChars: int = 2000):
        """Greedy pack under the 2000-character budget of
        browser/convertToLLMMessageService.ts:832-854 -> the '# APO Optimized Rules' block ('' if none)."""
        rules = self.getOptimizedRules()
        content, included = "", 0
        for r in rules:
            cand = content + ("\n" if content else "") + r
            if len(cand) > maxChars:
                break
            content, included = cand, included + 1
        if not content:
            return ""
        note = f" ({included}/{len(rules)} rules, budget limited)" if included < len(rules) else ""
        return f"\n\n# APO Optimized Rules{note}\n" + content

    # ---- queries
    def getLatestReport(self):
        return self._reports[-1] if self._reports else None

    def getPendingSuggestions(self):
        return [s for s in self._suggestions if s["status"] == "pending"]

    def getStats(self):
        """APO:1470-1508; avgFinalReward = mean over the 20 most recent traces by startTime desc
        (stable) with a non-null finalReward (APO:1478-1487) — 20 values, host side."""
        traces = [t for t in self._tc.getAllTraces() if t["summary"]["finalReward"] is not None]
        recent = sorted(traces, key=lambda t: -t["startTime"])[:20]
        acc = 0
        for t in recent:
            acc = acc + t["summary"]["finalReward"]
        last = self.getLatestReport()
        st = self._beamState
        return {"totalReports": len(self._reports), "totalSuggestions": len(self._suggestions),
                "appliedSuggestions": sum(1 for s in self._suggestions if s["status"] == "applied"),
                "rejectedSuggestions": sum(1 for s in self._suggestions if s["status"] == "rejected"),
                "activeSegments": len(self.getActiveSegments()),
                "optimizedSegments": sum(1 for s in self._segments if s["isActive"] and s["isOptimized"]),
                "lastAnalysisTime": last["generatedAt"] if last else None, "currentGoodRate": last["goodRate"] if last else None,
                "beamSearchActive": st is not None,                                  # APO:1502
                "beamCurrentRound": st["currentRound"] if st else None,
                "beamBestScore": st["historyBestScore"] if st and st["historyBestScore"] != -math.inf else None,
                "totalTextualGradients": len(self._textualGradients),
                "avgFinalReward": acc / len(recent) if recent else None}

    def getConfig(self):
        return dict(self._config)

    def setConfig(self, config):                                               # APO:1514-1526 (timers belong to the host application)
        self._config.update(config)
        self._saveConfig()
        self._fire(self._stateListeners)

    def getBeamState(self):
        return copy.deepcopy(self._beamState)

    def getTextualGradients(self, limit=None):                                 # newest first (APO:1534-1537)
        g = sorted(self._textualGradients, key=lambda t: -t["createdAt"])
        return g[:limit] if limit else g

    # ---- persistence (APO:336-413): same keys, same caps
    def _loadFromStorage(self):
        st = self._storage
        if not st:
            return
        try:
            if st.get(APO_CONFIG_KEY):
                self._config = {**DEFAULT_APO_CONFIG, **json.loads(st[APO_CONFIG_KEY])}
            if st.get(APO_STORAGE_KEY):
                data = json.loads(st[APO_STORAGE_KEY])
                self._reports, self._suggestions = data.get("reports") or [], data.get("suggestions") or []
            if st.get(APO_SEGMENTS_KEY):
                self._segments = json.loads(st[APO_SEGMENTS_KEY])
            if st.get(APO_BEAM_KEY):
                self._beamState = json.loads(st[APO_BEAM_KEY], parse_constant=_js_constant)
            if st.get(APO_GRADIENTS_KEY):
                self._textualGradients = json.loads(st[APO_GRADIENTS_KEY])
        except Exception as e:
            print("[APO] Failed to load from storage:", e)

    def _saveToStorage(self):
        if not self._dirty:
            return
        try:
            self._reports = self._reports[-MAX_REPORTS:]
            self._suggestions = self._suggestions[-MAX_SUGGESTIONS:]
            if self._storage is not None:
                self._storage[APO_STORAGE_KEY] = json.dumps({"reports": self._reports, "suggestions": self._suggestions})
                self._storage[APO_SEGMENTS_KEY] = json.dumps(self._segments)
                if self._beamState:
                    # JSON.stringify(-Infinity) is null: a never-scored beam reloads with historyBestScore null (APO:388-392)
                    self._storage[APO_BEAM_KEY] = json.dumps(_finite_or_none(self._beamState))
                if self._textualGradients:
                    self._textualGradients = self._textualGradients[-MAX_GRADIENTS:]
                    self._storage[APO_GRADIENTS_KEY] = json.dumps(self._textualGradients)
            self._dirty = False
        except Exception as e:
            print("[APO] Failed to save to storage:", e)

    def _saveConfig(self):
        try:
            if self._storage is not None:
                self._storage[APO_CONFIG_KEY] = json.dumps(self._config)
        except Exception:
            pass

    def dispose(self):                                                         # APO:1539-1542
        self._saveToStorage()

    # ---- periodic analysis (APO:453-475): the host application's timer calls this
    def _tryAutoAnalyze(self, now_ms=None):
        c = self._config
        if not c["enabled"] or not c["autoAnalyzeEnabled"]:
            return None
        stats = self._tc.getStats()
        if stats["totalTraces"] < c["minTracesForAnalysis"] or stats["totalFeedbacks"] < c["minFeedbacksForAnalysis"]:
            return None
        now_ms = time.time() * 1000.0 if now_ms is None else now_ms
        last = self.getLatestReport()
        if last and now_ms - last["generatedAt"] < c["autoAnalyzeIntervalMs"]:
            return None
        report = self.analyzePromptEffectiveness()
        if report["goodRate"] < 0.7 and c["uploadOptimizationsToServer"] and stats["totalFeedbacks"] >= 15:
            self.requestTextualGradient()
        return report

    def exportState(self):
        return json.dumps({"reports": self._reports, "suggestions": self._suggestions, "segments": self._segments,
                           "beamState": self._beamState, "config": self._config}, default=str)
