/*---------------------------------------------------------------------------------------------
 *  NEW FILE for src/vs/workbench/contrib/senweaver/electron-main/apoScoringMainService.ts
 *
 *  Main-process owner of the native addon (napi/apo_napi.c -> libapo_b200.so).  Registered in
 *  src/vs/code/electron-main/app.ts next to the other senweaver channels (app.ts:1258-1274), see
 *  ts/patches/app.ts.patch:
 *
 *      services.set(IApoScoringService, new SyncDescriptor(ApoScoringMainService));
 *      mainProcessElectronServer.registerChannel(APO_SCORING_CHANNEL,
 *          ProxyChannel.fromService(accessor.get(IApoScoringService), disposables));
 *
 *  The addon is loaded with a guarded dynamic import, like every optional native module of the
 *  IDE (platform/log/node/spdlogLog.ts:20-35); a failure only disables the fast path.
 *
 *  Threading: every addon call that touches the GPU is async work on the libuv pool, and the addon
 *  runs the jobs of one handle strictly in submission order (ticket FIFO, napi/apo_jobs.h), so
 *  overlapping IPC calls from several windows cannot race on the engine handle and an
 *  upload -> scoreResident sequence keeps its meaning without any promise chaining here.
 *--------------------------------------------------------------------------------------------*/
import { VSBuffer } from '../../../../base/common/buffer.js';
import { ApoResidentQuery, ApoScoreBlocks, ApoTupleBuffers, IApoScoringService } from '../common/apoScoringService.js';

type Blocks = { scores: ArrayBuffer; counts: ArrayBuffer; topk: ArrayBuffer; report: ArrayBuffer; candidates?: ArrayBuffer; candidateCorpus?: ArrayBuffer;
	candidateExtremes?: ArrayBuffer; candidateGroups?: ArrayBuffer; candidateSpread?: ArrayBuffer;
	candidatePairs?: ArrayBuffer; candidateGroupPairs?: ArrayBuffer };

interface ApoAddon {
	create(device: number): unknown | null;             // null when no H100 / library: never throws
	lastCreateError(): string;
	dimsUpload(handle: unknown, dims: ArrayBuffer, C: number, T: number, compact: boolean): Promise<void>;
	rolloutsUpload(handle: unknown, records: ArrayBuffer, rowBytes: number, C: number, T: number): Promise<void>;
	corpusUpload(handle: unknown, records: ArrayBuffer, idxBase: number): Promise<void>;
	corpusUploadJson(handle: unknown, utf8: ArrayBuffer, idxBase: number): Promise<number>;
	dimsTuples(handle: unknown, cap?: number): Promise<number>;
	recordGroupsUpload(handle: unknown, labels: ArrayBuffer, G: number): Promise<void>;
	candidateRefsUpload(handle: unknown, refs: ArrayBuffer): Promise<void>;
	scoreResident(handle: unknown, query: ApoResidentQuery): Promise<Blocks>;
	score(handle: unknown, dims: ArrayBuffer, C: number, T: number, corpus: ArrayBuffer | null, K: number, candidates?: boolean,
		candidateExtremes?: boolean, candidateGroups?: number, candidateSpread?: boolean,
		candidatePairs?: boolean, candidateGroupPairs?: number): Promise<Blocks>;
	scoreHostRecords(handle: unknown, records: ArrayBuffer, rowBytes: number, C: number, T: number, corpus: ArrayBuffer | null, K: number,
		candidates?: boolean, candidateCorpus?: boolean, candidateExtremes?: boolean, candidateGroups?: number, candidateSpread?: boolean,
		candidatePairs?: boolean, candidateGroupPairs?: number): Promise<Blocks>;
	/** Form D -> Form T on worker threads of the addon (no GPU): 3 bytes per evaluation instead of 36; null = not categorical. */
	encodeTuples(dims: ArrayBuffer, C: number, T: number, nthreads?: number): Promise<ApoTuples | null>;
	scoreHostTuples(handle: unknown, tuples: ApoTuples, C: number, T: number, corpus: ArrayBuffer | null, K: number, candidates?: boolean,
		candidateExtremes?: boolean, candidateGroups?: number, candidateSpread?: boolean,
		candidatePairs?: boolean, candidateGroupPairs?: number): Promise<Blocks>;
	rewardBatch(handle: unknown, records: ArrayBuffer): Promise<{ dims: ArrayBuffer; masks: ArrayBuffer; finals: ArrayBuffer }>;
	recordsFromJson(utf8: ArrayBuffer): ArrayBuffer | null;
}

/** Form T (include/apo_b200.h): 24-bit dictionary index per evaluation as two planes + the dictionary of distinct evaluations. */
interface ApoTuples { tl: ArrayBuffer; th: ArrayBuffer; tbookPc: ArrayBuffer; tbookPd: ArrayBuffer; codebook: ArrayBuffer; d2book: ArrayBuffer; nTuples: number }

const RECORD_BYTES = 32;

function ab(buf: VSBuffer): ArrayBuffer {
	const u8 = buf.buffer;
	return u8.buffer.slice(u8.byteOffset, u8.byteOffset + u8.byteLength) as ArrayBuffer;
}

function wrapBlocks(r: Blocks): ApoScoreBlocks {
	const out: ApoScoreBlocks = {
		scores: VSBuffer.wrap(new Uint8Array(r.scores)), counts: VSBuffer.wrap(new Uint8Array(r.counts)),
		topk: VSBuffer.wrap(new Uint8Array(r.topk)), report: VSBuffer.wrap(new Uint8Array(r.report)),
	};
	if (r.candidates) { out.candidates = VSBuffer.wrap(new Uint8Array(r.candidates)); }     // apo_candidate_report[C]
	if (r.candidateCorpus) { out.candidateCorpus = VSBuffer.wrap(new Uint8Array(r.candidateCorpus)); }     // apo_corpus_report[C]
	if (r.candidateExtremes) { out.candidateExtremes = VSBuffer.wrap(new Uint8Array(r.candidateExtremes)); }     // struct apo_candidate_extremes[C]
	if (r.candidateGroups) { out.candidateGroups = VSBuffer.wrap(new Uint8Array(r.candidateGroups)); }     // apo_group_score[C][G]
	if (r.candidateSpread) { out.candidateSpread = VSBuffer.wrap(new Uint8Array(r.candidateSpread)); }     // struct apo_candidate_spread[C]
	if (r.candidatePairs) { out.candidatePairs = VSBuffer.wrap(new Uint8Array(r.candidatePairs)); }     // struct apo_candidate_pair[C]
	if (r.candidateGroupPairs) { out.candidateGroupPairs = VSBuffer.wrap(new Uint8Array(r.candidateGroupPairs)); }     // struct apo_candidate_pair[C][G]
	return out;
}

interface PendingReward {
	records: Uint8Array;
	resolve: (r: { dims: VSBuffer; masks: VSBuffer; finals: VSBuffer }) => void;
	reject: (e: unknown) => void;
}

export class ApoScoringMainService implements IApoScoringService {
	readonly _serviceBrand: undefined;
	private _addon: ApoAddon | undefined;
	private _handle: unknown;
	private readonly _ready: Promise<void>;
	private _pendingRewards: PendingReward[] = [];

	constructor() {
		this._ready = this._load();
	}

	private async _load(): Promise<void> {
		try {
			const mod = await import('apo_b200.node' as string);      // unpacked from the asar by build/gulpfile.vscode.js:315
			const addon = (mod.default ?? mod) as ApoAddon;
			const handle = addon.create(0);                            // null when no H100 is visible: there is no CPU fallback
			if (handle === null || handle === undefined) {
				console.warn('[APO] native scoring engine unavailable:', addon.lastCreateError());
				return;
			}
			this._addon = addon;
			this._handle = handle;
		} catch (e) {
			console.warn('[APO] native scoring engine unavailable:', e instanceof Error ? e.message : String(e));
			this._addon = undefined;
		}
	}

	private async _need(): Promise<ApoAddon> {
		await this._ready;
		if (!this._addon) { throw new Error('apo_b200 addon not loaded'); }
		return this._addon;
	}

	async isAvailable(): Promise<boolean> {
		await this._ready;
		return !!this._addon;
	}

	/** Single-trace rewards arrive one by one (endTrace / recordUserFeedback, TCS:413, 547): the requests of one tick are
	 *  concatenated into ONE apo_reward_batch call and the result is sliced back per caller. */
	async rewardBatch(records: VSBuffer) {
		await this._need();
		return new Promise<{ dims: VSBuffer; masks: VSBuffer; finals: VSBuffer }>((resolve, reject) => {
			this._pendingRewards.push({ records: records.buffer, resolve, reject });
			if (this._pendingRewards.length === 1) { queueMicrotask(() => this._flushRewards()); }
		});
	}

	private _flushRewards(): void {
		const batch = this._pendingRewards;
		this._pendingRewards = [];
		if (!this._addon || batch.length === 0) { return; }
		const total = batch.reduce((n, p) => n + p.records.byteLength, 0);
		const all = new Uint8Array(total);
		let off = 0;
		for (const p of batch) { all.set(p.records, off); off += p.records.byteLength; }
		this._addon.rewardBatch(this._handle, all.buffer as ArrayBuffer).then(r => {
			let rec = 0;
			for (const p of batch) {
				const n = p.records.byteLength / RECORD_BYTES;
				p.resolve({
					dims: VSBuffer.wrap(new Uint8Array(r.dims, rec * 72, n * 72)),
					masks: VSBuffer.wrap(new Uint8Array(r.masks, rec * 4, n * 4)),
					finals: VSBuffer.wrap(new Uint8Array(r.finals, rec * 8, n * 8)),
				});
				rec += n;
			}
		}, e => { for (const p of batch) { p.reject(e); } });
	}

	async recordsFromJson(persisted: string): Promise<VSBuffer> {
		const addon = await this._need();
		const out = addon.recordsFromJson(ab(VSBuffer.fromString(persisted)));
		if (!out) { throw new Error('malformed trace JSON'); }
		return VSBuffer.wrap(new Uint8Array(out));
	}

	// ---- resident path ------------------------------------------------------------------------
	async dimsUpload(dims: VSBuffer, C: number, T: number, compact?: boolean): Promise<void> {
		return (await this._need()).dimsUpload(this._handle, ab(dims), C, T, !!compact);
	}

	async rolloutsUpload(records: VSBuffer, rowBytes: 32 | 16, C: number, T: number): Promise<void> {
		return (await this._need()).rolloutsUpload(this._handle, ab(records), rowBytes, C, T);
	}

	async corpusUpload(records: VSBuffer, idxBase?: number): Promise<void> {
		return (await this._need()).corpusUpload(this._handle, ab(records), idxBase ?? 0);
	}

	async corpusUploadJson(persisted: string, idxBase?: number): Promise<number> {
		return (await this._need()).corpusUploadJson(this._handle, ab(VSBuffer.fromString(persisted)), idxBase ?? 0);
	}

	async dimsTuples(cap?: number): Promise<number> {
		return (await this._need()).dimsTuples(this._handle, cap);
	}

	async recordGroupsUpload(labels: VSBuffer, G: number): Promise<void> {
		return (await this._need()).recordGroupsUpload(this._handle, ab(labels), G);
	}

	async candidateRefsUpload(refs: VSBuffer): Promise<void> {
		return (await this._need()).candidateRefsUpload(this._handle, ab(refs));
	}

	async scoreResident(query: ApoResidentQuery): Promise<ApoScoreBlocks> {
		return wrapBlocks(await (await this._need()).scoreResident(this._handle, query));
	}

	// ---- one-shot path ------------------------------------------------------------------------
	async score(dims: VSBuffer, C: number, T: number, corpus: VSBuffer | undefined, K: number, candidates?: boolean,
		candidateExtremes?: boolean, candidateGroups?: number, candidateSpread?: boolean, candidatePairs?: boolean,
		candidateGroupPairs?: number): Promise<ApoScoreBlocks> {
		return wrapBlocks(await (await this._need()).score(this._handle, ab(dims), C, T, corpus ? ab(corpus) : null, K, !!candidates,
			!!candidateExtremes, candidateGroups ?? 0, !!candidateSpread, !!candidatePairs,
			candidateGroupPairs ?? 0));
	}

	/** fp32 evaluations -> Form T (3 bytes per evaluation + the dictionary of distinct evaluations); undefined when the tensor is not
	 *  categorical enough.  Encoding reads the 36-byte rows twice on the addon's worker threads — several times the cost of sending
	 *  them over PCIe once — so it pays for evaluations that are scored MORE THAN ONCE (beam rounds over the same rollouts, weight
	 *  sweeps), kept, or shipped between processes; a one-shot score() of fp32 rows stays the cheaper call. */
	async encodeTuples(dims: VSBuffer, C: number, T: number): Promise<ApoTupleBuffers | undefined> {
		const t = await (await this._need()).encodeTuples(ab(dims), C, T);
		if (!t) { return undefined; }
		const w = (b: ArrayBuffer) => VSBuffer.wrap(new Uint8Array(b));
		return { tl: w(t.tl), th: w(t.th), tbookPc: w(t.tbookPc), tbookPd: w(t.tbookPd), codebook: w(t.codebook), d2book: w(t.d2book), nTuples: t.nTuples };
	}

	/** Same result as score() on the tensor the tuples were encoded from; 12x fewer bytes over IPC and PCIe. */
	async scoreTuples(t: ApoTupleBuffers, C: number, T: number, corpus: VSBuffer | undefined, K: number, candidates?: boolean,
		candidateExtremes?: boolean, candidateGroups?: number, candidateSpread?: boolean, candidatePairs?: boolean,
		candidateGroupPairs?: number): Promise<ApoScoreBlocks> {
		const raw: ApoTuples = { tl: ab(t.tl), th: ab(t.th), tbookPc: ab(t.tbookPc), tbookPd: ab(t.tbookPd), codebook: ab(t.codebook), d2book: ab(t.d2book), nTuples: t.nTuples };
		return wrapBlocks(await (await this._need()).scoreHostTuples(this._handle, raw, C, T, corpus ? ab(corpus) : null, K, !!candidates,
			!!candidateExtremes, candidateGroups ?? 0, !!candidateSpread, !!candidatePairs,
			candidateGroupPairs ?? 0));
	}

	async scoreHostRecords(records: VSBuffer, rowBytes: 32 | 16, C: number, T: number, corpus: VSBuffer | undefined, K: number,
		candidates?: boolean, candidateCorpus?: boolean, candidateExtremes?: boolean, candidateGroups?: number,
		candidateSpread?: boolean, candidatePairs?: boolean, candidateGroupPairs?: number): Promise<ApoScoreBlocks> {
		return wrapBlocks(await (await this._need()).scoreHostRecords(this._handle, ab(records), rowBytes, C, T, corpus ? ab(corpus) : null, K, !!candidates,
			!!candidateCorpus, !!candidateExtremes, candidateGroups ?? 0, !!candidateSpread, !!candidatePairs,
			candidateGroupPairs ?? 0));
	}
}
