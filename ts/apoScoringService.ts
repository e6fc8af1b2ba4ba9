/*---------------------------------------------------------------------------------------------
 *  NEW FILE for src/vs/workbench/contrib/senweaver/common/apoScoringService.ts
 *
 *  Common-layer contract + renderer-side proxy of the GPU scoring engine.  The `common`
 *  layer may not load native code (eslint.config.js:94-111), so this file only declares the
 *  service and builds a ProxyChannel client; the implementation lives in the main process
 *  (apoScoringMainService.ts), exactly like the metrics service of the reference
 *  (common/metricsService.ts:25-50 / electron-main/metricsMainService.ts:35).
 *
 *  This file cannot be compiled in the engine's build image (no tsc / node); it is the
 *  reference-side binding INTEGRATION.md describes.
 *--------------------------------------------------------------------------------------------*/
import { VSBuffer } from '../../../../base/common/buffer.js';
import { ProxyChannel } from '../../../../base/parts/ipc/common/ipc.js';
import { createDecorator } from '../../../../platform/instantiation/common/instantiation.js';
import { registerSingleton, InstantiationType } from '../../../../platform/instantiation/common/extensions.js';
import { IMainProcessService } from '../../../../platform/ipc/common/mainProcessService.js';

export const APO_SCORING_CHANNEL = 'senweaver-channel-apoScoring';

/** Raw result blocks; layouts are those of include/apo_b200.h (see traceRecordCodec.ts). */
export interface ApoScoreBlocks {
	scores: VSBuffer;   // float64[C]  (-Infinity: candidate without a non-null evaluation)
	counts: VSBuffer;   // uint64[C]
	topk: VSBuffer;     // int32[K]    score desc, ties -> lower index
	report: VSBuffer;   // struct apo_corpus_report (784 bytes)
	candidates?: VSBuffer;   // apo_candidate_report[C] (376 bytes each, candidateReportCodec.ts); only when the call asked for it
	candidateCorpus?: VSBuffer;   // apo_corpus_report[C] (784 bytes each, decodeCandidateCorpusReport); rollout records only, when asked for
	candidateExtremes?: VSBuffer;   // struct apo_candidate_extremes[C] (1032 bytes each, decodeCandidateExtremes); only when asked for
	candidateGroups?: VSBuffer;   // apo_group_score[C][G] (56 bytes each, decodeCandidateGroups); only when asked for
	candidateSpread?: VSBuffer;   // struct apo_candidate_spread[C] (88 bytes each, decodeCandidateSpread); only when asked for
	candidatePairs?: VSBuffer;   // struct apo_candidate_pair[C] (128 bytes each, decodeCandidatePairs); only when asked for
	candidateGroupPairs?: VSBuffer;   // struct apo_candidate_pair[C][G] (128 bytes each, decodeCandidateGroupPairs); only when asked for
}

/** Form T of a float32[C][T][9] tensor (include/apo_b200.h): tl uint16[C][T] | th uint8[C][T] = the 24-bit dictionary index of every
 *  evaluation; tbookPc uint32[n] / tbookPd uint16[n] = the n distinct evaluations as Form P pairs; codebook uint32[8][256], d2book
 *  uint32[4096] = the fp32 bit patterns the codes stand for. */
export interface ApoTupleBuffers {
	tl: VSBuffer; th: VSBuffer; tbookPc: VSBuffer; tbookPd: VSBuffer; codebook: VSBuffer; d2book: VSBuffer; nTuples: number;
}

/** What a resident scoring call selects (apo_score_opts of include/apo_b200.h). */
export interface ApoResidentQuery {
	C: number;              // candidates uploaded with dimsUpload / rolloutsUpload
	K: number;              // beam width (APOConfig.beamWidth, APO:288)
	source?: 0 | 1 | 2;     // 0 = dims (Form D / Form Q), 1 = per-(candidate, trace) records, 2 = Form T built by dimsTuples
	corpus?: 0 | 1;         // also build the corpus report from the uploaded corpus
	candidates?: 0 | 1;     // also build the per-candidate breakdown (ApoScoreBlocks.candidates)
	candidateCorpus?: 0 | 1;   // source 1 only: also build every candidate's corpus report (ApoScoreBlocks.candidateCorpus)
	candidateExtremes?: 0 | 1;   // also list every candidate's 32 lowest- and highest-reward rollouts (ApoScoreBlocks.candidateExtremes)
	candidateGroups?: number;   // G of the uploaded record groups: also split every candidate's rollouts by group (ApoScoreBlocks.candidateGroups)
	candidateSpread?: 0 | 1;   // also build every candidate's reward spread (ApoScoreBlocks.candidateSpread)
	candidatePairs?: 0 | 1;   // also compare every candidate with its candidateRefsUpload reference (ApoScoreBlocks.candidatePairs)
	candidateGroupPairs?: number;   // G of the uploaded record groups: also make that comparison per group (ApoScoreBlocks.candidateGroupPairs)
	first?: number;         // window [first, first + count) of the trace axis; count 0 = to the end
	count?: number;
}

export interface IApoScoringService {
	readonly _serviceBrand: undefined;
	/** false when the addon or an H100 is unavailable: callers keep their state untouched and warn. */
	isAvailable(): Promise<boolean>;
	/** TraceCollectorService._computeRewardSignals for n packed records (apo_reward_batch).  Calls made in the same tick
	 *  are coalesced into one engine call by the main-process service. */
	rewardBatch(records: VSBuffer): Promise<{ dims: VSBuffer; masks: VSBuffer; finals: VSBuffer }>;
	/** The string stored under 'senweaver.traceCollector.data' -> packed Form R records (apo_records_from_json):
	 *  lets a stored corpus reach the engine without materialising ConversationTrace objects. */
	recordsFromJson(persisted: string): Promise<VSBuffer>;

	// ---- resident path: uploaded once, scored many times (only the result block crosses PCIe again)
	/** float32[C][T][9], NaN = dimension absent.  compact: keep the lossless 14-byte layout on the device. */
	dimsUpload(dims: VSBuffer, C: number, T: number, compact?: boolean): Promise<void>;
	/** [C][T] trace records, 32-byte apo_record or 16-byte apo_record16 rows; dims are derived on the device (TCS:668-763). */
	rolloutsUpload(records: VSBuffer, rowBytes: 32 | 16, C: number, T: number): Promise<void>;
	/** The traces _buildReport walks (APO:498-625), one 32-byte record each; idxBase = index of the first one. */
	corpusUpload(records: VSBuffer, idxBase?: number): Promise<void>;
	/** Same from the persisted JSON string; resolves to the number of traces. */
	corpusUploadJson(persisted: string, idxBase?: number): Promise<number>;
	/** Build resident Form T (3 bytes per evaluation, source 2) on the device from the uploaded dims (apo_dims_tuples); resolves
	 *  to the number of dictionary entries.  Rejects, leaving no Form T, when the dims hold more than cap distinct evaluations
	 *  (default and maximum 16777215) or are not categorical.  Pays when the same dims are scored more than once. */
	dimsTuples(cap?: number): Promise<number>;
	/** One uint8 label per rollout index, each < G <= 64 (a chat mode, a task category, a held-out split): calls that pass
	 *  candidateGroups = G then split every candidate's rollouts by these groups.  An empty buffer releases them. */
	recordGroupsUpload(labels: VSBuffer, G: number): Promise<void>;
	/** One uint32 per candidate: the index of its reference (its parent), or 0xFFFFFFFF for none.  Calls of C candidates that
	 *  pass candidatePairs then compare every candidate with its reference on the rollouts both were scored on.  An empty buffer
	 *  releases them. */
	candidateRefsUpload(refs: VSBuffer): Promise<void>;
	scoreResident(query: ApoResidentQuery): Promise<ApoScoreBlocks>;

	// ---- one-shot path: host buffers streamed through the device, nothing stays resident
	/** dims: float32[C][T][9] (pass C = 1, T = 4 of NaN for report-only calls).
	 *  candidates: also return the per-candidate breakdown (ApoScoreBlocks.candidates), here and on the other one-shot calls;
	 *  candidateExtremes: also return every candidate's 32 lowest- and highest-reward rollouts (ApoScoreBlocks.candidateExtremes);
	 *  candidateGroups: the G of recordGroupsUpload, also return every candidate's scores per record group (ApoScoreBlocks.candidateGroups);
	 *  candidateSpread: also return every candidate's reward spread (ApoScoreBlocks.candidateSpread);
	 *  candidatePairs: also compare every candidate with its reference (ApoScoreBlocks.candidatePairs);
	 *  candidateGroupPairs: the G of recordGroupsUpload, also make that comparison per record group (ApoScoreBlocks.candidateGroupPairs). */
	score(dims: VSBuffer, C: number, T: number, corpus: VSBuffer | undefined, K: number, candidates?: boolean,
		candidateExtremes?: boolean, candidateGroups?: number, candidateSpread?: boolean, candidatePairs?: boolean,
		candidateGroupPairs?: number): Promise<ApoScoreBlocks>;
	/** [C][T] trace records (the IDE's own representation): 2.2x fewer PCIe bytes than fp32 dims with 16-byte rows.
	 *  candidateCorpus: also return the corpus report of every candidate's records (ApoScoreBlocks.candidateCorpus). */
	scoreHostRecords(records: VSBuffer, rowBytes: 32 | 16, C: number, T: number, corpus: VSBuffer | undefined, K: number, candidates?: boolean,
		candidateCorpus?: boolean, candidateExtremes?: boolean, candidateGroups?: number, candidateSpread?: boolean, candidatePairs?: boolean,
		candidateGroupPairs?: number): Promise<ApoScoreBlocks>;
	/** fp32 evaluations -> Form T (include/apo_b200.h): a 24-bit dictionary index per evaluation (3 bytes instead of 36) + the
	 *  dictionary of distinct evaluations.  For evaluations that are scored more than once, kept, or moved between processes. */
	encodeTuples(dims: VSBuffer, C: number, T: number): Promise<ApoTupleBuffers | undefined>;
	scoreTuples(tuples: ApoTupleBuffers, C: number, T: number, corpus: VSBuffer | undefined, K: number, candidates?: boolean,
		candidateExtremes?: boolean, candidateGroups?: number, candidateSpread?: boolean, candidatePairs?: boolean,
		candidateGroupPairs?: number): Promise<ApoScoreBlocks>;
}

export const IApoScoringService = createDecorator<IApoScoringService>('senweaverApoScoringService');

/** Renderer-side client: everything that crosses the channel is async (metricsService.ts:47). */
export class ApoScoringService implements IApoScoringService {
	readonly _serviceBrand: undefined;
	private readonly _proxy: IApoScoringService;

	constructor(@IMainProcessService mainProcessService: IMainProcessService) {
		this._proxy = ProxyChannel.toService<IApoScoringService>(mainProcessService.getChannel(APO_SCORING_CHANNEL));
	}

	isAvailable(): Promise<boolean> { return this._proxy.isAvailable(); }
	rewardBatch(records: VSBuffer) { return this._proxy.rewardBatch(records); }
	recordsFromJson(persisted: string) { return this._proxy.recordsFromJson(persisted); }
	dimsUpload(dims: VSBuffer, C: number, T: number, compact?: boolean) { return this._proxy.dimsUpload(dims, C, T, compact); }
	rolloutsUpload(records: VSBuffer, rowBytes: 32 | 16, C: number, T: number) { return this._proxy.rolloutsUpload(records, rowBytes, C, T); }
	corpusUpload(records: VSBuffer, idxBase?: number) { return this._proxy.corpusUpload(records, idxBase); }
	corpusUploadJson(persisted: string, idxBase?: number) { return this._proxy.corpusUploadJson(persisted, idxBase); }
	dimsTuples(cap?: number) { return this._proxy.dimsTuples(cap); }
	recordGroupsUpload(labels: VSBuffer, G: number) { return this._proxy.recordGroupsUpload(labels, G); }
	candidateRefsUpload(refs: VSBuffer) { return this._proxy.candidateRefsUpload(refs); }
	scoreResident(query: ApoResidentQuery) { return this._proxy.scoreResident(query); }
	// A call without group scores, spreads, pairs or group pairs sends the channel the same arguments as before those options existed.
	score(dims: VSBuffer, C: number, T: number, corpus: VSBuffer | undefined, K: number, candidates?: boolean, candidateExtremes?: boolean,
		candidateGroups?: number, candidateSpread?: boolean, candidatePairs?: boolean, candidateGroupPairs?: number) {
		if (candidateGroupPairs) {
			return this._proxy.score(dims, C, T, corpus, K, candidates, candidateExtremes, candidateGroups ?? 0, !!candidateSpread, !!candidatePairs,
				candidateGroupPairs);
		}
		if (candidatePairs) { return this._proxy.score(dims, C, T, corpus, K, candidates, candidateExtremes, candidateGroups ?? 0, !!candidateSpread, true); }
		if (candidateSpread) { return this._proxy.score(dims, C, T, corpus, K, candidates, candidateExtremes, candidateGroups ?? 0, true); }
		if (candidateGroups) { return this._proxy.score(dims, C, T, corpus, K, candidates, candidateExtremes, candidateGroups); }
		return this._proxy.score(dims, C, T, corpus, K, candidates, candidateExtremes);
	}
	scoreHostRecords(records: VSBuffer, rowBytes: 32 | 16, C: number, T: number, corpus: VSBuffer | undefined, K: number, candidates?: boolean,
		candidateCorpus?: boolean, candidateExtremes?: boolean, candidateGroups?: number, candidateSpread?: boolean, candidatePairs?: boolean,
		candidateGroupPairs?: number) {
		if (candidateGroupPairs) {
			return this._proxy.scoreHostRecords(records, rowBytes, C, T, corpus, K, candidates, candidateCorpus, candidateExtremes, candidateGroups ?? 0,
				!!candidateSpread, !!candidatePairs, candidateGroupPairs);
		}
		if (candidatePairs) {
			return this._proxy.scoreHostRecords(records, rowBytes, C, T, corpus, K, candidates, candidateCorpus, candidateExtremes, candidateGroups ?? 0,
				!!candidateSpread, true);
		}
		if (candidateSpread) {
			return this._proxy.scoreHostRecords(records, rowBytes, C, T, corpus, K, candidates, candidateCorpus, candidateExtremes, candidateGroups ?? 0, true);
		}
		if (candidateGroups) { return this._proxy.scoreHostRecords(records, rowBytes, C, T, corpus, K, candidates, candidateCorpus, candidateExtremes, candidateGroups); }
		return this._proxy.scoreHostRecords(records, rowBytes, C, T, corpus, K, candidates, candidateCorpus, candidateExtremes);
	}
	encodeTuples(dims: VSBuffer, C: number, T: number) { return this._proxy.encodeTuples(dims, C, T); }
	scoreTuples(tuples: ApoTupleBuffers, C: number, T: number, corpus: VSBuffer | undefined, K: number, candidates?: boolean,
		candidateExtremes?: boolean, candidateGroups?: number, candidateSpread?: boolean, candidatePairs?: boolean, candidateGroupPairs?: number) {
		if (candidateGroupPairs) {
			return this._proxy.scoreTuples(tuples, C, T, corpus, K, candidates, candidateExtremes, candidateGroups ?? 0, !!candidateSpread, !!candidatePairs,
				candidateGroupPairs);
		}
		if (candidatePairs) {
			return this._proxy.scoreTuples(tuples, C, T, corpus, K, candidates, candidateExtremes, candidateGroups ?? 0, !!candidateSpread, true);
		}
		if (candidateSpread) { return this._proxy.scoreTuples(tuples, C, T, corpus, K, candidates, candidateExtremes, candidateGroups ?? 0, true); }
		if (candidateGroups) { return this._proxy.scoreTuples(tuples, C, T, corpus, K, candidates, candidateExtremes, candidateGroups); }
		return this._proxy.scoreTuples(tuples, C, T, corpus, K, candidates, candidateExtremes);
	}
}

registerSingleton(IApoScoringService, ApoScoringService, InstantiationType.Delayed);
