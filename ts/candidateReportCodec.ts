/*---------------------------------------------------------------------------------------------
 *  NEW FILE for src/vs/workbench/contrib/senweaver/common/candidateReportCodec.ts
 *
 *  Decoder of the per-candidate breakdown (ApoScoreBlocks.candidates): apo_candidate_report[C] of
 *  include/apo_b200.h, the numbers _buildReport computes for the corpus (APO:498-625) answered for
 *  every beam candidate — feedback tallies, goodRate, avgReward (== the candidate's score),
 *  rewardByDimension with the dim-low / suggestion flags (APO:575/591/802/819), and the first three
 *  rollouts of the candidate whose feedback was 'bad'.  The beam loop's critique step
 *  (_buildTextualGradientPrompt, APO:918-962) can name what a parent lost on from this.
 *
 *  Also the decoder of the per-candidate corpus reports (ApoScoreBlocks.candidateCorpus): apo_corpus_report[C], the whole
 *  corpus report of each candidate's rollout records (problem patterns, byMode, tool totals included), decoded by
 *  traceRecordCodec's decodeCorpusReport.
 *
 *  And the decoder of the per-candidate extremes (ApoScoreBlocks.candidateExtremes): struct apo_candidate_extremes[C], the
 *  32 lowest- and 32 highest-reward rollouts of each candidate with their finalRewards — the sample runs the critique prompt
 *  is built from (APO:918-962, 1003-1007).
 *
 *  And the decoder of the per-candidate group scores (ApoScoreBlocks.candidateGroups): apo_group_score[C][G], each candidate's
 *  tallies and exact mean reward on the rollouts of every record group (a chat mode, a task category, a held-out split).
 *
 *  And the decoder of the per-candidate reward spreads (ApoScoreBlocks.candidateSpread): struct apo_candidate_spread[C], each
 *  candidate's exact reward sums and the variance, standard deviation and standard error of its mean: the scale against which
 *  the gap between two candidates' scores can be read.
 *
 *  And the decoder of the paired comparisons (ApoScoreBlocks.candidatePairs): struct apo_candidate_pair[C], each candidate
 *  against its reference on the rollouts both were scored on: wins, losses, ties, the exact paired sums and the mean reward
 *  difference with its standard error.  decodeCandidateGroupPairs reads the same record per (candidate, group) of a
 *  candidateGroupPairs block (struct apo_candidate_pair[C][G]): that comparison on the rollouts of each record group.
 *
 *  The byte offsets below are pinned to the C structs by tests/test_napi_candidates.py, tests/test_candidate_corpus_cpu.py,
 *  tests/test_napi_candidate_extremes.py, tests/test_candidate_groups_cpu.py, tests/test_candidate_spread_cpu.py and
 *  tests/test_candidate_pairs_cpu.py.
 *--------------------------------------------------------------------------------------------*/
import { VSBuffer } from '../../../../base/common/buffer.js';
import { CorpusReportNumbers, DIM_NAMES, decodeCorpusReport } from './traceRecordCodec.js';

const CANDIDATE_REPORT_BYTES = 376;
const OFF_TOTAL = 0;
const OFF_GOOD = 8;
const OFF_BAD = 16;
const OFF_NONE = 24;
const OFF_GOOD_RATE = 32;
const OFF_WITH_REWARD = 40;
const OFF_REWARD_SUM = 48;
const OFF_AVG_REWARD = 56;
const OFF_DIM = 64;
const DIMSTAT_BYTES = 32;
const OFF_BAD_EXAMPLES = 352;
// inside one apo_dimstat (sum at 0)
const DIM_COUNT = 8;
const DIM_AVG = 16;
const DIM_LOW_FLAG = 24;
const DIM_LOW_SEVERITY = 25;
const DIM_SUGG_FLAG = 26;
const DIM_SUGG_PRIORITY = 27;

export interface CandidateReportNumbers {
	candidate: number;
	total: number; goodFeedbackCount: number; badFeedbackCount: number; noFeedbackCount: number; goodRate: number;
	withReward: number; rewardSum: number; avgReward: number | null;
	rewardByDimension: Record<string, { sum: number; count: number; avg: number; low: 'medium' | 'high' | null; suggest: 'medium' | 'high' | null }>;
	badExamples: number[];                 // rollout indices (the candidate's record axis), ascending
}

const u64 = (v: DataView, o: number) => Number(v.getBigUint64(o, true));

/** Number of reports in a candidates block. */
export function candidateReportCount(buf: VSBuffer): number {
	return Math.floor(buf.byteLength / CANDIDATE_REPORT_BYTES);
}

/** Report c of a candidates block (ApoScoreBlocks.candidates). */
export function decodeCandidateReport(buf: VSBuffer, c: number): CandidateReportNumbers {
	const base = c * CANDIDATE_REPORT_BYTES;
	if (c < 0 || base + CANDIDATE_REPORT_BYTES > buf.byteLength) { throw new RangeError(`candidate ${c} outside the block`); }
	const v = new DataView(buf.buffer.buffer, buf.buffer.byteOffset + base, CANDIDATE_REPORT_BYTES);
	const rewardByDimension: CandidateReportNumbers['rewardByDimension'] = {};
	DIM_NAMES.forEach((name, i) => {
		const o = OFF_DIM + DIMSTAT_BYTES * i, count = u64(v, o + DIM_COUNT);
		if (count) {
			rewardByDimension[name] = {
				sum: v.getFloat64(o, true), count, avg: v.getFloat64(o + DIM_AVG, true),
				low: v.getUint8(o + DIM_LOW_FLAG) ? (v.getUint8(o + DIM_LOW_SEVERITY) === 2 ? 'high' : 'medium') : null,      // APO:575, 591
				suggest: v.getUint8(o + DIM_SUGG_FLAG) ? (v.getUint8(o + DIM_SUGG_PRIORITY) === 2 ? 'high' : 'medium') : null, // APO:802, 819
			};
		}
	});
	const badExamples = [0, 1, 2].map(k => Number(v.getBigInt64(OFF_BAD_EXAMPLES + 8 * k, true))).filter(x => x >= 0);
	const withReward = u64(v, OFF_WITH_REWARD);
	return {
		candidate: c, total: u64(v, OFF_TOTAL), goodFeedbackCount: u64(v, OFF_GOOD), badFeedbackCount: u64(v, OFF_BAD),
		noFeedbackCount: u64(v, OFF_NONE), goodRate: v.getFloat64(OFF_GOOD_RATE, true), withReward,
		rewardSum: v.getFloat64(OFF_REWARD_SUM, true), avgReward: withReward ? v.getFloat64(OFF_AVG_REWARD, true) : null,
		rewardByDimension, badExamples,
	};
}

const CORPUS_REPORT_BYTES = 784;         // sizeof(apo_corpus_report)

/** Number of reports in a candidateCorpus block. */
export function candidateCorpusReportCount(buf: VSBuffer): number {
	return Math.floor(buf.byteLength / CORPUS_REPORT_BYTES);
}

/** Corpus report of candidate c from a candidateCorpus block (ApoScoreBlocks.candidateCorpus); pattern examples are rollout
 *  indices (absolute positions on the candidate's record axis). */
export function decodeCandidateCorpusReport(buf: VSBuffer, c: number): CorpusReportNumbers {
	const base = c * CORPUS_REPORT_BYTES;
	if (c < 0 || base + CORPUS_REPORT_BYTES > buf.byteLength) { throw new RangeError(`candidate ${c} outside the block`); }
	return decodeCorpusReport(buf.slice(base, base + CORPUS_REPORT_BYTES));
}

const EXTREMES_BYTES = 1032;             // sizeof(struct apo_candidate_extremes)
const EXTREMES_N = 32;
const OFF_EXT_N = 0;
const OFF_LOWEST = 8;
const OFF_LOWEST_REWARD = 264;
const OFF_HIGHEST = 520;
const OFF_HIGHEST_REWARD = 776;

export interface CandidateExtremes {
	candidate: number;
	lowestRollouts: { index: number; finalReward: number }[];    // finalReward ascending, ties -> lower index
	highestRollouts: { index: number; finalReward: number }[];   // finalReward descending, ties -> lower index
}

/** Number of entries in a candidateExtremes block. */
export function candidateExtremesCount(buf: VSBuffer): number {
	return Math.floor(buf.byteLength / EXTREMES_BYTES);
}

/** The lists of candidate c from a candidateExtremes block (ApoScoreBlocks.candidateExtremes); indices are rollout positions on
 *  the candidate's record axis, rewards the finalRewards the scoring call summed. */
export function decodeCandidateExtremes(buf: VSBuffer, c: number): CandidateExtremes {
	const base = c * EXTREMES_BYTES;
	if (c < 0 || base + EXTREMES_BYTES > buf.byteLength) { throw new RangeError(`candidate ${c} outside the block`); }
	const v = new DataView(buf.buffer.buffer, buf.buffer.byteOffset + base, EXTREMES_BYTES);
	const n = Math.min(u64(v, OFF_EXT_N), EXTREMES_N);
	const list = (offIdx: number, offRew: number) => Array.from({ length: n }, (_, i) => ({
		index: Number(v.getBigInt64(offIdx + 8 * i, true)), finalReward: v.getFloat64(offRew + 8 * i, true),
	}));
	return { candidate: c, lowestRollouts: list(OFF_LOWEST, OFF_LOWEST_REWARD), highestRollouts: list(OFF_HIGHEST, OFF_HIGHEST_REWARD) };
}

const GROUP_SCORE_BYTES = 56;            // sizeof(apo_group_score)
const OFF_GRP_TOTAL = 0;
const OFF_GRP_GOOD = 8;
const OFF_GRP_BAD = 16;
const OFF_GRP_GOOD_RATE = 24;
const OFF_GRP_WITH_REWARD = 32;
const OFF_GRP_REWARD_SUM = 40;
const OFF_GRP_AVG_REWARD = 48;

export interface GroupScore {
	totalRollouts: number;
	goodFeedbackCount: number;
	badFeedbackCount: number;
	goodRate: number;
	withReward: number;
	rewardSum: number;
	avgReward: number | null;   // null when none of the group's rollouts has a reward
}

/** The group scores of a candidateGroups block (ApoScoreBlocks.candidateGroups) of C candidates and G groups: [C][G]. */
export function decodeCandidateGroups(buf: VSBuffer, C: number, G: number): GroupScore[][] {
	if (C < 0 || G < 1 || C * G * GROUP_SCORE_BYTES > buf.byteLength) { throw new RangeError(`${C} x ${G} group scores do not fit the block`); }
	const v = new DataView(buf.buffer.buffer, buf.buffer.byteOffset, C * G * GROUP_SCORE_BYTES);
	return Array.from({ length: C }, (_, c) => Array.from({ length: G }, (_, g) => {
		const o = (c * G + g) * GROUP_SCORE_BYTES;
		const withReward = u64(v, o + OFF_GRP_WITH_REWARD);
		return {
			totalRollouts: u64(v, o + OFF_GRP_TOTAL), goodFeedbackCount: u64(v, o + OFF_GRP_GOOD), badFeedbackCount: u64(v, o + OFF_GRP_BAD),
			goodRate: v.getFloat64(o + OFF_GRP_GOOD_RATE, true), withReward, rewardSum: v.getFloat64(o + OFF_GRP_REWARD_SUM, true),
			avgReward: withReward === 0 ? null : v.getFloat64(o + OFF_GRP_AVG_REWARD, true),
		};
	}));
}

const CANDIDATE_SPREAD_BYTES = 88;       // sizeof(struct apo_candidate_spread)
const OFF_SPR_N = 0;
const OFF_SPR_SUM_LO = 8;
const OFF_SPR_SUM_HI = 16;
const OFF_SPR_SUM_SQ = 24;
const OFF_SPR_MEAN = 48;
const OFF_SPR_REWARD_SUM_SQ = 56;
const OFF_SPR_VARIANCE = 64;
const OFF_SPR_STD_DEV = 72;
const OFF_SPR_STD_ERR = 80;

export interface CandidateSpread {
	candidate: number;
	n: number;                 // rewarded rollouts (== counts[c])
	sum: bigint;               // exact sum of rint(finalReward * 2^52) over them
	sumSq: bigint;             // exact sum of its squares
	mean: number | null;       // == the candidate's score; null when n == 0
	rewardSumSq: number;       // sumSq * 2^-104, rounded once
	variance: number | null;   // sample variance of the rewards; null when n < 2
	stdDev: number | null;
	stdErr: number | null;     // standard error of mean
}

/** The reward spreads of a candidateSpread block (ApoScoreBlocks.candidateSpread) of C candidates. */
export function decodeCandidateSpread(buf: VSBuffer, C: number): CandidateSpread[] {
	if (C < 0 || C * CANDIDATE_SPREAD_BYTES > buf.byteLength) { throw new RangeError(`${C} candidate spreads do not fit the block`); }
	return Array.from({ length: C }, (_, c) => {
		const v = new DataView(buf.buffer.buffer, buf.buffer.byteOffset + c * CANDIDATE_SPREAD_BYTES, CANDIDATE_SPREAD_BYTES);
		const n = u64(v, OFF_SPR_N);
		const f = (o: number) => v.getFloat64(o, true);
		const sumSq = v.getBigUint64(OFF_SPR_SUM_SQ, true) | (v.getBigUint64(OFF_SPR_SUM_SQ + 8, true) << 64n) |
			(v.getBigUint64(OFF_SPR_SUM_SQ + 16, true) << 128n);
		return {
			candidate: c, n, sum: (v.getBigInt64(OFF_SPR_SUM_HI, true) << 64n) | v.getBigUint64(OFF_SPR_SUM_LO, true), sumSq,
			mean: n === 0 ? null : f(OFF_SPR_MEAN), rewardSumSq: f(OFF_SPR_REWARD_SUM_SQ),
			variance: n < 2 ? null : f(OFF_SPR_VARIANCE), stdDev: n < 2 ? null : f(OFF_SPR_STD_DEV), stdErr: n < 2 ? null : f(OFF_SPR_STD_ERR),
		};
	});
}

const CANDIDATE_PAIR_BYTES = 128;        // sizeof(struct apo_candidate_pair)
const PAIR_NONE = 0xFFFFFFFF;
const OFF_PR_REF = 0;
const OFF_PR_N = 8;
const OFF_PR_WINS = 16;
const OFF_PR_LOSSES = 24;
const OFF_PR_TIES = 32;
const OFF_PR_CAND_ONLY = 40;
const OFF_PR_REF_ONLY = 48;
const OFF_PR_SUM_LO = 56;
const OFF_PR_SUM_HI = 64;
const OFF_PR_SUM_SQ = 72;
const OFF_PR_MEAN_DIFF = 96;
const OFF_PR_VARIANCE = 104;
const OFF_PR_STD_DEV = 112;
const OFF_PR_STD_ERR = 120;

export interface CandidatePair {
	candidate: number;
	reference: number | null;  // null: the candidate had no reference
	n: number;                 // positions where both have a reward
	wins: number; losses: number; ties: number;
	candOnly: number;          // positions where only the candidate has a reward
	refOnly: number;           // positions where only the reference has a reward
	sum: bigint;               // exact sum of d = rint(fr_c * 2^52) - rint(fr_r * 2^52) over the n positions
	sumSq: bigint;             // exact sum of d^2
	meanDiff: number | null;   // mean reward difference; null when n == 0
	variance: number | null;   // sample variance of the differences; null when n < 2
	stdDev: number | null;
	stdErr: number | null;     // standard error of meanDiff
}

/** The paired comparisons of a candidatePairs block (ApoScoreBlocks.candidatePairs) of C candidates. */
export function decodeCandidatePairs(buf: VSBuffer, C: number): CandidatePair[] {
	if (C < 0 || C * CANDIDATE_PAIR_BYTES > buf.byteLength) { throw new RangeError(`${C} candidate pairs do not fit the block`); }
	return Array.from({ length: C }, (_, c) => decodePair(buf, c * CANDIDATE_PAIR_BYTES, c));
}

/** The paired comparisons per record group of a candidateGroupPairs block (ApoScoreBlocks.candidateGroupPairs) of C candidates
 *  and G groups: out[c][g] is candidate c against its reference on the rollouts of group g. */
export function decodeCandidateGroupPairs(buf: VSBuffer, C: number, G: number): CandidatePair[][] {
	if (C < 0 || G < 1 || C * G * CANDIDATE_PAIR_BYTES > buf.byteLength) {
		throw new RangeError(`${C} x ${G} candidate group pairs do not fit the block`);
	}
	return Array.from({ length: C }, (_, c) => Array.from({ length: G }, (_, g) => decodePair(buf, (c * G + g) * CANDIDATE_PAIR_BYTES, c)));
}

/** One struct apo_candidate_pair at byte offset off of the block: candidate c against its reference. */
function decodePair(buf: VSBuffer, off: number, c: number): CandidatePair {
	const v = new DataView(buf.buffer.buffer, buf.buffer.byteOffset + off, CANDIDATE_PAIR_BYTES);
	const ref = v.getUint32(OFF_PR_REF, true);
	const n = u64(v, OFF_PR_N);
	const f = (o: number) => v.getFloat64(o, true);
	const sumSq = v.getBigUint64(OFF_PR_SUM_SQ, true) | (v.getBigUint64(OFF_PR_SUM_SQ + 8, true) << 64n) |
		(v.getBigUint64(OFF_PR_SUM_SQ + 16, true) << 128n);
	return {
		candidate: c, reference: ref === PAIR_NONE ? null : ref, n, wins: u64(v, OFF_PR_WINS), losses: u64(v, OFF_PR_LOSSES),
		ties: u64(v, OFF_PR_TIES), candOnly: u64(v, OFF_PR_CAND_ONLY), refOnly: u64(v, OFF_PR_REF_ONLY),
		sum: (v.getBigInt64(OFF_PR_SUM_HI, true) << 64n) | v.getBigUint64(OFF_PR_SUM_LO, true), sumSq,
		meanDiff: n === 0 ? null : f(OFF_PR_MEAN_DIFF),
		variance: n < 2 ? null : f(OFF_PR_VARIANCE), stdDev: n < 2 ? null : f(OFF_PR_STD_DEV), stdErr: n < 2 ? null : f(OFF_PR_STD_ERR),
	};
}
