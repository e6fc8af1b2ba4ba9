/*
 * apo_b200.h — C ABI of the H100-native (sm_90a) APO scoring engine (libapo_b200.so).
 *
 * Drop-in boundary for ONE hot path of senweaver/senweaver-ide: the 9-dimension reward
 * -> finalReward aggregation, the 6-pattern problem detector and the top-K beam
 * selection behind APOService / TraceCollectorService.  Plain C types only; no C++,
 * torch or CUDA types cross this boundary.  Every entry point below names the reference
 * code it replaces:
 *   TCS = src/vs/workbench/contrib/senweaver/common/traceCollectorService.ts
 *   APO = src/vs/workbench/contrib/senweaver/common/apoService.ts
 *
 * Conventions (reference error behaviour, TCS:438, APO:1211-1214: never throw into the
 * caller): every function returns 0 on success or a negative APO_E_* code; the message
 * is available from apo_last_error().  Nothing is retained from host pointers after a
 * call returns.  A handle is not re-entrant (one in-flight call per handle); distinct
 * handles are independent.  There is NO CPU fallback: without a CUDA device every
 * compute entry point fails with APO_E_CUDA.
 */
#ifndef APO_B200_H
#define APO_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define APO_ABI_VERSION 2
#define APO_NDIM  9   /* reward dimensions, push order of TCS:679..762 */
#define APO_NPAT  6   /* problem patterns, APO:643-770 */
#define APO_NMODE 5   /* 0 no metadata ('unknown', APO:632), 1 normal, 2 agent, 3 gather, 4 designer */

#define APO_OK          0
#define APO_E_ARG      -1   /* bad argument                       */
#define APO_E_CUDA     -2   /* CUDA runtime / no device           */
#define APO_E_STATE    -3   /* call order (nothing uploaded, ...) */
#define APO_E_NOMEM    -4
#define APO_E_NCCL     -5

/* Form R — one trace-summary record = the fields of ConversationTrace.summary that the
 * path reads (TCS:94-108) + endTime (TCS:87) + metadata.chatMode (TCS:91) + the span
 * counts of TCS:752-753 / APO:667-669,733.  32 bytes, little endian. */
typedef struct apo_record {
	uint8_t  feedback;   /* 0 null, 1 'good', 2 'bad' */
	uint8_t  flags;      /* APO_F_* */
	uint8_t  mode;       /* chat mode code, see APO_NMODE */
	uint8_t  durClass;   /* APO_DC_*: what the path asks of totalToolDurationMs, decided in binary64 by the encoder; 0 = derive from toolDurMs */
	uint16_t userMsgs;   /* # user_message spans */
	uint16_t asstMsgs;   /* # assistant_message spans */
	uint32_t toolCalls, toolSucc, toolFail, llmCalls, tokens;
	float    toolDurMs;  /* totalToolDurationMs rounded to binary32 (the value itself is only read when durClass is 0) */
} apo_record;
/* The reference compares totalToolDurationMs (a JS double: fractional performance.now() deltas) with 0 and 15000 and its
 * per-call average with 1000 / 3000 / 10000 in binary64 (TCS:721-728, APO:754).  A binary32 copy can land on the other side of
 * a threshold, so encoders that hold the double (the TypeScript codec, the JSON ingest, apo_duration_class) store the four
 * comparison results here; records without them (durClass == 0: synthetic generators, hand-built records) are scored from
 * toolDurMs, which is exact whenever the duration is representable in binary32. */
#define APO_DC_SET     0x80u  /* the bits below are valid                                           */
#define APO_DC_LEVEL   0x03u  /* how many of avg > 1000, avg > 3000, avg > 10000 hold (TCS:724-727) */
#define APO_DC_POS     0x04u  /* totalToolDurationMs > 0 (TCS:721)                                  */
#define APO_DC_SLOW    0x08u  /* totalToolDurationMs > 15000 (APO:754)                              */
#define APO_F_ERRORS   0x01u  /* summary.hasErrors                                   */
#define APO_F_ENDED    0x02u  /* endTime set                                         */
#define APO_F_VALID    0x08u  /* summary.finalReward !== null (TCS:606, APO:550)     */
#define APO_F_FAILSPAN 0x10u  /* a tool_call span with toolSuccess===false exists    */

/* Form R16 — the same record packed into 16 bytes for transport over PCIe / storage.
 * Saturating fields keep every output of the path unchanged: userMsgs/asstMsgs only meet
 * thresholds <= 9 (TCS:756-761, APO:734), llmCalls saturates the reward at n >= 8 (TCS:735),
 * tokens only meets thresholds <= 30000 (TCS:741-747, APO:693).  toolSucc is implied by
 * toolCalls - toolFail (they are incremented together, TCS:505-510).  Records that do not
 * satisfy that, or whose toolCalls/toolFail exceed 65535, are rejected by apo_record_pack16
 * and must travel as Form R. */
typedef struct apo_record16 {
	uint16_t hdr;        /* bits 0-1 feedback, 2 hasErrors, 3 ended, 4 valid, 5 failspan, 6-8 mode */
	uint8_t  userMsgs, asstMsgs;
	uint16_t toolCalls, toolFail;
	uint8_t  llmCalls, durClass;
	uint16_t tokens;
	float    toolDurMs;
} apo_record16;

typedef struct apo_pattern {      /* one of the six patterns of APO:635-773 */
	uint64_t count;               /* frequency                              */
	uint8_t  flag;                /* emitted (count >= minimum)             */
	uint8_t  severity;            /* 0 low, 1 medium, 2 high                */
	uint8_t  pad[6];
	int64_t  examples[3];         /* first 3 matching record indices (corpus order), -1 = none */
} apo_pattern;

typedef struct apo_dimstat {      /* APO:556-568 + rules APO:575,591,802,819 */
	double   sum; uint64_t count; double avg;
	uint8_t  low_flag, low_severity, sugg_flag, sugg_priority;
	uint8_t  pad[4];
} apo_dimstat;

typedef struct apo_corpus_report { /* numeric content of APO._buildReport + TCS.getStats */
	uint64_t total, good, bad, none;          /* APO:509-516 */
	double   goodRate;                        /* APO:546-547 */
	uint64_t byMode[APO_NMODE][3];            /* total, good, bad (APO:519-525) */
	double   byModeGoodRate[APO_NMODE];       /* APO:541-544 */
	uint64_t withReward;                      /* APO:550 */
	double   rewardSum;
	double   avgReward;                       /* NaN = null */
	apo_dimstat dim[APO_NDIM];
	apo_pattern pat[APO_NPAT];
	uint64_t toolCalls, toolSucc, toolFail;   /* TCS:603-605 */
	double   toolSuccessRate;                 /* TCS:624, NaN = null */
} apo_corpus_report;

typedef struct apo_timing {       /* device time of the stages of the last apo_score*, ms (CUDA events) */
	float reward_ms;              /* K1 reward9 / reward9_raw                 */
	float corpus_ms;              /* K2 detect6 (+ fused finalize at 1 rank)  */
	float allreduce_ms;           /* ncclAllReduce of the packed partials     */
	float finalize_ms;            /* K3 segmented sum + radix top-K (>1 rank) */
	float total_ms;               /* first launch -> last kernel end          */
	uint32_t launches;            /* kernels launched by the call             */
	uint32_t pad;
	float join_wait_ms;           /* peer-memory join: publish -> every rank arrived (includes rank skew), device timer */
	float join_reduce_ms;         /* peer-memory join: NVLink reads + sum of the peers' partial vectors                 */
	float tail_finalize_ms;       /* K3 in the finalising CTA: segmented sum + report + radix top-K (device timer)      */
	float tail_publish_ms;        /* result block written to the caller's page-locked buffer + accumulators re-armed    */
} apo_timing;
/* The *_ms stage fields come from CUDA events, which are recorded only for calls that stream >= 64 MB or set
 * APO_SCORE_TIMING (a small call is launch-bound and every event costs it ~1 us); launches and the join_* fields
 * (device-side timer) are always filled. */

typedef struct apo_engine apo_engine;

/* ---- lifecycle ------------------------------------------------------------------ */
int  apo_abi_version(void);
/* One engine drives one GPU (one process per GPU).  device = CUDA ordinal. */
int  apo_create(int device, apo_engine **out);
void apo_destroy(apo_engine *e);
/* Message of the last failure on this engine (e == NULL: last apo_create failure). */
const char *apo_last_error(const apo_engine *e);
/* Launch all work on this CUDA stream (a cudaStream_t passed as an integer); 0 = the
 * engine's own stream.  Lets a host harness bracket calls with its own events. */
int  apo_set_stream(apo_engine *e, uint64_t cuda_stream);
/* Replace the TCS:766-776 weights (default = reference values). */
int  apo_set_weights(apo_engine *e, const double w[APO_NDIM]);
/* Experiment / test switches of one handle (initial value: the environment variables APO_NO_FUSE, APO_FORCE_FUSE,
 * APO_NO_STAGING, APO_JOIN_NCCL, APO_NO_TWIN, APO_NO_TWIN_T, APO_TWIN_T, APO_NO_TWIN_T2 read once at apo_create).  Results are identical for
 * every setting. */
#define APO_TUNE_NO_FUSE     0x1u  /* corpus scan / finalisation as stand-alone launches                         */
#define APO_TUNE_FORCE_FUSE  0x2u  /* corpus scan inside the scoring launch even when it cannot hide behind it   */
#define APO_TUNE_NO_STAGING  0x4u  /* pageable host buffers straight to cudaMemcpy (no threaded pinned staging)  */
#define APO_TUNE_NCCL_JOIN   0x8u  /* join shards with ncclAllReduce + k_finalize instead of the peer-memory join */
#define APO_TUNE_NO_TWIN     0x10u /* no Form Q / W copy of a loaded Form D tensor is built or read: resident Form D runs K1 */
#define APO_TUNE_NO_TWIN_T   0x20u /* no Form T copy of a loaded Form D tensor is built or read: the Form Q / W copy as without it */
#define APO_TUNE_TWIN_T      0x40u /* loads build the Form T copy whatever the tensor's size (tests, A/B runs on small tensors) */
#define APO_TUNE_NO_TWIN_T2  0x80u /* no exception list of the Form T copy is built or read: the copy is read at 3 B per evaluation */
int  apo_set_tuning(apo_engine *e, uint32_t flags);
int  apo_get_weights(const apo_engine *e, double w[APO_NDIM]);

/* ---- single-trace path: TraceCollectorService._computeRewardSignals (TCS:668-788) --
 * dims: n x 9 binary64, NaN where the dimension is not pushed; masks: 9-bit presence;
 * finals: finalReward, NaN where it stays null (VALID flag clear). Computed on the GPU. */
int apo_reward_batch(apo_engine *e, const apo_record *recs, uint64_t n,
                     double *dims, uint32_t *masks, double *finals);
int apo_reward_one(apo_engine *e, const apo_record *rec, double dims[APO_NDIM],
                   uint32_t *mask, double *final_reward);

/* ---- corpus = the T trace records APOService._buildReport walks (APO:498-625) ------
 * idx_base = global index of recs[0] (shard offset); example indices are global. */
int apo_corpus_upload(apo_engine *e, const apo_record *recs, uint64_t T, uint64_t idx_base);
int apo_corpus_generate(apo_engine *e, uint64_t seed, uint64_t t0, uint64_t T, uint32_t agent_permille);
int apo_corpus_download(apo_engine *e, apo_record *out, uint64_t first, uint64_t n);

/* ---- ingest: the reference's persisted traces -> Form R (SURVEY 8f rank 1) ----------
 * json = the value TraceCollectorService._saveToStorage writes under
 * 'senweaver.traceCollector.data' (TCS:296-359): JSON.stringify(ConversationTrace[]).  One record
 * per trace in array order: counters from summary (TCS:94-108), ENDED from a truthy endTime
 * (TCS:686), VALID from finalReward !== null (TCS:606), mode from metadata.chatMode (TCS:91),
 * userMsgs/asstMsgs/FAILSPAN counted from the spans (TCS:752-753, APO:667-669).
 * apo_records_from_json needs no engine and no GPU (format code only): returns the number of
 * traces in the array (records beyond cap are counted, not written) or APO_E_ARG on malformed
 * input, with the byte offset of the failure in *err_pos (may be NULL).
 * apo_corpus_upload_json = parse + apo_corpus_upload(idx_base); *n_records (may be NULL) gets T.
 * Note: the engine derives finalReward from the record.  A trace whose counters kept moving after
 * its reward was set (endTraceForThread leaves the trace active, TCS:420-425) re-scores from the
 * later counters; callers that need the stored value keep the record snapshot taken at scoring
 * time (what the TraceCollectorService mirror does) and upload those with apo_corpus_upload. */
int64_t apo_records_from_json(const char *json, uint64_t len, apo_record *out, uint64_t cap, uint64_t *err_pos);
int apo_corpus_upload_json(apo_engine *e, const char *json, uint64_t len, uint64_t idx_base, uint64_t *n_records);

/* ---- candidate x record evaluations ------------------------------------------------
 * Form D: fp32 dims[C][T][9], NaN = dimension absent, all-NaN = finalReward null.  Domain: every
 * evaluation's finalReward within [-512, 512) (the reference range is [-1,1], TCS:36), so that the
 * sums are exact fixed point; a Form D / Q / P evaluation outside it (a finalReward of 512 or more,
 * below -512, +-inf) fails the scoring call with APO_E_ARG.
 * Form R: one apo_record per (candidate, record); dims derived on device (TCS:668-763).
 * apo_dims_upload and apo_dims_generate also build a Form Q copy of the tensor (see below) when its evaluations are
 * categorical and at least 4 GiB of device memory stays free beside the copy; otherwise, quietly, they keep Form D alone.
 * When no coded dimension (every one but d2) takes more than 15 values (true for dims produced by TCS:668-763) and 4 GiB
 * also stay free beside the Form Q planes and one more 8-byte word per evaluation, the copy is kept as Form W instead: per
 * evaluation eight 4-bit codes (15 = absent) and the fp32 tool_success_rate bits (one NaN pattern = absent), 8 B.
 * Resident Form D calls with variant 0 and a window starting on a multiple of 8 then read the copy through K1q (8 B or 14 B
 * instead of 36 B per evaluation); other variants and windows read the fp32 tensor through K1.  The results are the same
 * either way.  The fp32 tensor stays loaded (apo_dims_layout 1, apo_dims_download); the copy goes with the next load or
 * attach, and whenever an engine allocation would otherwise fail for lack of device memory.  apo_dims_attach never
 * builds one: the caller owns that memory and may change it.
 * Beside a Form W copy (or a Form Q one with <= 15 values per coded dimension) a tensor of at least 2^26 evaluations also gets
 * a Form T copy (3 B per evaluation: indices into a dictionary of its distinct evaluations, built as apo_dims_tuples builds
 * resident Form T) when it holds at most 2^20 distinct evaluations, the 24576 most frequent cover at least 3/4 of them, and
 * 4 GiB stay free beside it; the same calls then read that copy through K1t whenever the weights keep every entry inside
 * (-2, 2), else the Form W / Q copy.  It is not resident Form T (APO_SRC_TUPLES never sees it) and goes with the Form W / Q
 * copy.  APO_TUNE_NO_TWIN_T turns it off, APO_TUNE_TWIN_T builds it at any size.
 * When at most 1/64 of the evaluations have a dictionary index of 2^16 or more, the copy also holds a list of those
 * evaluations, and the calls read 2 B per evaluation (the low 16 bits of every index) and correct the listed ones; with at
 * most 2^16 distinct evaluations the list is empty.  APO_TUNE_NO_TWIN_T2 at the load builds no list, set later it keeps the
 * calls at 3 B per evaluation. */
int apo_dims_upload(apo_engine *e, const float *dims, uint32_t C, uint64_t T);
int apo_dims_generate(apo_engine *e, uint64_t seed, uint32_t c0, uint32_t C, uint64_t t0, uint64_t T,
                      uint32_t agent_permille);
int apo_dims_download(apo_engine *e, float *out, uint32_t c, uint64_t first, uint64_t n);
/* Form Q — compact resident layout (csrc/apo_compact.cu): 8 one-byte codebook indices + the
 * fp32 tool_success_rate + a 2-byte presence index per evaluation (14 B instead of 36 B), lossless.  Available when every
 * dimension except d2 takes <= 255 distinct values (true for dims produced by TCS:668-763).
 * apo_dims_compact transcodes the loaded Form D in place (the fp32 copy is released; when the Form Q copy
 * built at load is held, it becomes the tensor without a second transcode; a Form W copy is released first);
 * the *_compact generate/upload variants never materialise the full fp32 tensor.  When the data
 * is not categorical they return APO_E_STATE: apo_dims_compact keeps the loaded Form D usable, the
 * streaming variants leave nothing loaded.  Scores, counts, top-K and the integer partial sums are
 * bit-identical between the two layouts. */
int apo_dims_compact(apo_engine *e);
int apo_dims_generate_compact(apo_engine *e, uint64_t seed, uint32_t c0, uint32_t C, uint64_t t0, uint64_t T,
                              uint32_t agent_permille);
int apo_dims_upload_compact(apo_engine *e, const float *dims, uint32_t C, uint64_t T);
/* 0 nothing loaded, 1 Form D (fp32), 2 Form Q (compact) */
int apo_dims_layout(const apo_engine *e);
/* Use a caller-owned device buffer (row pitch in evals, >= T rounded up to 4; 16-byte
 * aligned base).  The engine never frees it. */
int apo_dims_attach(apo_engine *e, uint64_t device_ptr, uint32_t C, uint64_t T, uint64_t pitch_evals);
int apo_rollouts_upload(apo_engine *e, const apo_record *recs, uint32_t C, uint64_t T);
int apo_rollouts_generate(apo_engine *e, uint64_t seed, uint32_t c0, uint32_t C, uint64_t t0, uint64_t T,
                          uint32_t agent_permille);
int apo_rollouts_download(apo_engine *e, apo_record *out, uint32_t c, uint64_t first, uint64_t n);
/* Packed rollouts (Form R16, 16 B per evaluation): same scoring source APO_SRC_ROLLOUTS. */
int apo_rollouts16_upload(apo_engine *e, const apo_record16 *recs, uint32_t C, uint64_t T);
int apo_rollouts16_generate(apo_engine *e, uint64_t seed, uint32_t c0, uint32_t C, uint64_t t0, uint64_t T,
                            uint32_t agent_permille);
int apo_rollouts16_download(apo_engine *e, apo_record16 *out, uint32_t c, uint64_t first, uint64_t n);
/* Host-side format helpers (no device work).  pack returns APO_E_ARG and the index of the first
 * unrepresentable record in *bad (may be NULL). */
/* durClass of a trace from the binary64 duration and the call count, exactly as TCS:721-728 / APO:754 compare them. */
uint8_t apo_duration_class(double totalToolDurationMs, uint32_t totalToolCalls);
int apo_record_pack16(const apo_record *in, uint64_t n, apo_record16 *out, uint64_t *bad);
int apo_record_unpack16(const apo_record16 *in, uint64_t n, apo_record *out);

/* ---- scoring: score[c] = mean_t finalReward[c,t] (APO:550-553 per candidate), top-K
 * (score desc, ties -> lower index; replaces the server-side beam selection consumed at
 * APO:1138-1166) and, when a corpus is loaded and APO_SCORE_CORPUS is set, the corpus
 * report (APO:498-625, 635-773; TCS:596-626). */
#define APO_SRC_DIMS      0u
#define APO_SRC_ROLLOUTS  1u
#define APO_SRC_TUPLES    2u   /* resident Form T (apo_tuples_upload) */
#define APO_SCORE_CORPUS  0x1u   /* also run the 6-pattern scan over the corpus */
#define APO_SCORE_RECIP   0x2u   /* finalReward = ws * (1/tw) from a LUT instead of ws / tw (<= 1 ulp apart) */
#define APO_SCORE_TIMING  0x4u   /* record the per-stage CUDA events of apo_timing also for a small call */
#define APO_SCORE_CANDIDATES 0x8u /* also build the per-candidate breakdown (apo_candidate_reports) */
#define APO_SCORE_CANDIDATE_CORPUS 0x10u /* also build the corpus report of every candidate's rollout records (apo_candidate_corpus_reports) */
typedef struct apo_score_opts {
	uint32_t K;          /* beam width (top-K), 0..min(C, 16384) */
	uint32_t source;     /* APO_SRC_* */
	uint32_t flags;      /* APO_SCORE_* */
	uint32_t variant;    /* kernel variant, 0 = default (tuning / A-B only) */
	uint64_t first;      /* window [first, first+count) of the record axis, first % 4 == 0 (% 8 for Form Q / T); */
	uint64_t count;      /* count == 0 -> all records */
} apo_score_opts;
/* scores[C] (-inf when a candidate has no non-null evaluation), counts[C], topk[K];
 * any output pointer may be NULL. */
int apo_score(apo_engine *e, const apo_score_opts *o, double *scores, uint64_t *counts,
              int32_t *topk, apo_corpus_report *report);
/* Chunked form of apo_score for evaluation sets that exceed device memory (BASELINE
 * configs[4]: 1024 x 100M = 3.7 TB): begin zeroes the accumulators for C_total candidates;
 * each accumulate streams the currently loaded dims/rollouts (a chunk of candidates and/or
 * a window of records) into candidates [cand_offset, cand_offset + C_loaded); finish runs the
 * corpus scan, the cross-rank join and the top-K over all C_total.  apo_score ==
 * begin + one accumulate + finish.  finish may be called repeatedly within one session: the
 * candidate accumulators are exact integers that only ever grow by later accumulate calls, so
 * new records (a window that was not scored yet) can be added as they arrive and the ranking
 * refreshed without rescanning the old ones (incremental scoring). */
int apo_score_begin(apo_engine *e, uint32_t C_total);
int apo_score_accumulate(apo_engine *e, const apo_score_opts *o, uint32_t cand_offset);
int apo_score_finish(apo_engine *e, const apo_score_opts *o, double *scores, uint64_t *counts,
                     int32_t *topk, apo_corpus_report *report);
/* End to end from host memory without keeping the evaluations resident: streams
 * dims[C][T][9] through a double-buffered device window (H2D overlapped with K1). */
int apo_score_host(apo_engine *e, const apo_score_opts *o, const float *dims, uint32_t C, uint64_t T,
                   double *scores, uint64_t *counts, int32_t *topk, apo_corpus_report *report);
/* Same for per-(candidate, record) rollouts in host memory: row_bytes = 32 (apo_record) or
 * 16 (apo_record16); recs is [C][T] rows.  Dims are derived on the device (TCS:668-763). */
int apo_score_host_records(apo_engine *e, const apo_score_opts *o, const void *recs, uint32_t row_bytes,
                           uint32_t C, uint64_t T, double *scores, uint64_t *counts, int32_t *topk,
                           apo_corpus_report *report);
/* Form Q as a wire format — the same call for callers that hold the evaluations in the compact layout in host memory:
 * three planes [C][T] (q8: 8 one-byte codes per evaluation, d2: fp32 tool_success_rate, li: 2-byte presence index = 14 B
 * per evaluation instead of 36) + the codebook (8 x 256 fp32 bit patterns, 0xFFFFFFFF = unused) that assigns the codes.
 * apo_compact_encode_host builds them from Form D on the host (two passes on nthreads threads; APO_E_STATE when a coded
 * dimension has more than 255 distinct values); apo_dims_compact_download / apo_dims_codebook export a resident Form Q
 * tensor.  Results are bit-identical to scoring the Form D tensor.  The codebook must be the one that assigned the planes'
 * codes: this call has no per-evaluation pass to check them, and a code naming an empty slot is scored as a present 0.0. */
int apo_compact_encode_host(const float *dims, uint32_t C, uint64_t T, uint64_t *q8, float *d2, uint16_t *li,
                            uint32_t *codebook /* [8*256] */, int nthreads);
int apo_dims_compact_download(apo_engine *e, uint64_t *q8, float *d2, uint16_t *li, uint32_t c, uint64_t first, uint64_t n);
int apo_dims_codebook(apo_engine *e, uint32_t *codebook /* [8*256] */);
int apo_score_host_compact(apo_engine *e, const apo_score_opts *o, const uint64_t *q8, const float *d2, const uint16_t *li,
                           const uint32_t *codebook, uint32_t C, uint64_t T, double *scores, uint64_t *counts, int32_t *topk,
                           apo_corpus_report *report);
/* Form P — the tightest lossless wire format (6 B per evaluation): pc = eight 4-bit codes in a uint32 (dimension order
 * 0,1,3,4,5,6,7,8; 15 = absent), pd = 12-bit index of the tool_success_rate value into d2book (4095 = absent), both [C][T].
 * Needs <= 15 distinct values per coded dimension and <= 4095 distinct tool_success_rate values (APO_E_STATE otherwise:
 * fall back to Form Q / Form D); dims produced by TCS:668-763 always qualify.  The device expands every window to Form Q
 * (k_unpack_p) right behind its H2D copy and scores it with K1q: same integers, 2.3x fewer PCIe bytes than Form Q.
 * Both codebooks travel with the planes (empty slots 0xFFFFFFFF): an evaluation whose code names an empty or NaN codebook
 * slot, or whose tool_success_rate index names an empty or NaN d2book slot, fails the call with APO_E_ARG. */
int apo_packed_encode_host(const float *dims, uint32_t C, uint64_t T, uint32_t *pc, uint16_t *pd,
                           uint32_t *codebook /* [8*256] */, uint32_t *d2book /* [4096] fp32 bit patterns */, int nthreads);
/* Export of a resident Form Q tensor in Form P (rows of candidate c) and the tool_success_rate table that goes with it
 * (the codebook is apo_dims_codebook's). */
int apo_dims_packed_download(apo_engine *e, uint32_t *pc, uint16_t *pd, uint32_t c, uint64_t first, uint64_t n);
int apo_dims_d2book(apo_engine *e, uint32_t *d2book /* [4096] */);
int apo_score_host_packed(apo_engine *e, const apo_score_opts *o, const uint32_t *pc, const uint16_t *pd, const uint32_t *codebook,
                          const uint32_t *d2book, uint32_t C, uint64_t T, double *scores, uint64_t *counts, int32_t *topk,
                          apo_corpus_report *report);
/* Form T — evaluations as dictionary indices (3 B per evaluation; csrc/apo_tuple.cu).  The nine dimensions of an evaluation are
 * functions of a few small counters (TCS:668-763), so a tensor of C x T evaluations holds only 10^5..10^6 DISTINCT ones.  tbook =
 * those, as Form P pairs (tbook_pc[i], tbook_pd[i]), most frequent first; every evaluation is the 24-bit index of its entry, kept
 * as a 16-bit plane tl and an 8-bit plane th, both [C][T].  Per scoring call the device evaluates finalReward once per ENTRY
 * (TCS:777-787, the operations of K1q) and K1t sums table entries per candidate: the integers are those of every other layout.
 * apo_tuple_encode_host builds the planes and the dictionary from Form P planes (two passes on nthreads threads); *n_tuples
 * receives the number of distinct evaluations; APO_E_STATE when that exceeds cap (<= 16777215 = APO_TUPLES_MAX) — keep Form P then.
 * apo_score_host_tuples streams the planes from host memory (as apo_score_host_packed does for Form P);
 * apo_tuples_upload makes them resident: apo_score / apo_score_accumulate with source APO_SRC_TUPLES then read 3 B per evaluation.
 * An index >= n_tuples in the planes, or a dictionary entry whose finalReward is not within (-2, 2) or that names an empty or
 * NaN slot of the codebook or of d2book, fails the call with APO_E_ARG.  Entries are checked whether or not an evaluation
 * names them. */
#define APO_TUPLES_MAX 16777215u
int apo_tuple_encode_host(const uint32_t *pc, const uint16_t *pd, uint32_t C, uint64_t T, uint16_t *tl, uint8_t *th,
                          uint32_t *tbook_pc, uint16_t *tbook_pd, uint32_t cap, uint32_t *n_tuples, int nthreads);
int apo_score_host_tuples(apo_engine *e, const apo_score_opts *o, const uint16_t *tl, const uint8_t *th, const uint32_t *tbook_pc,
                          const uint16_t *tbook_pd, uint32_t n_tuples, const uint32_t *codebook, const uint32_t *d2book,
                          uint32_t C, uint64_t T, double *scores, uint64_t *counts, int32_t *topk, apo_corpus_report *report);
int apo_tuples_upload(apo_engine *e, const uint16_t *tl, const uint8_t *th, const uint32_t *tbook_pc, const uint16_t *tbook_pd,
                      uint32_t n_tuples, const uint32_t *codebook, const uint32_t *d2book, uint32_t C, uint64_t T);
/* Form T built on the device from the loaded evaluations, without a host round trip.  It leaves the engine exactly as
 * apo_tuples_upload would with the planes, dictionary and n_tuples that apo_tuple_encode_host makes of this tensor's Form P
 * planes, and with the codebook and d2book that go with them (the tensor's own: apo_dims_codebook / apo_dims_d2book of its
 * Form Q layout).  Dictionary order: most frequent first, ties by key (code word | d2book index << 32) ascending; the bytes
 * are the same for every grid.  It reads the Form W copy that apo_dims_upload / apo_dims_generate keep of categorical dims, or
 * a Form Q layout or copy whose coded dimensions take <= 15 values each.  Afterwards source APO_SRC_TUPLES scores the result;
 * the loaded dims, their copy and their scoring are untouched, and the tuples stay loaded, independent of later dims loads,
 * until the next apo_tuples_upload or apo_dims_tuples.  The build is rank-local: each shard gets its own dictionary.
 * cap is clamped to APO_TUPLES_MAX.  APO_E_STATE, with nothing built, when: no dims are loaded; Form D is loaded without a
 * copy (APO_TUNE_NO_TWIN, apo_dims_attach, too little device memory at load: call apo_dims_compact first); a coded
 * dimension takes 16 or more values; tool_success_rate takes more than 4095 values; the evaluations hold more than cap
 * distinct ones (*n_tuples then receives a lower bound greater than cap, as from apo_tuple_encode_host).  APO_E_NOMEM when
 * the build's own allocations released the copy it reads.  After any failure no Form T is loaded; the dims are untouched.
 * Device scratch of the build (a hash table sized from min(cap, C*T), ~16 B per possible entry) is released on return. */
int apo_dims_tuples(apo_engine *e, uint32_t cap, uint32_t *n_tuples);
/* Rows of the resident Form T tensor (built or uploaded): tl / th of candidate c, records [first, first + n). */
int apo_tuples_download(apo_engine *e, uint16_t *tl, uint8_t *th, uint32_t c, uint64_t first, uint64_t n);
/* Its dictionary and codebooks.  *n_tuples always receives n; the entries are written only when cap >= n (APO_E_ARG
 * otherwise). */
int apo_tuples_book(apo_engine *e, uint32_t *tbook_pc, uint16_t *tbook_pd, uint32_t cap,
                    uint32_t *codebook /* [8*256] */, uint32_t *d2book /* [4096] */, uint32_t *n_tuples);
/* Host buffers for the streaming calls and the uploads.  Any host pointer is accepted: pageable memory (malloc, a JS
 * ArrayBuffer, numpy) is gathered chunk by chunk into pinned staging buffers by a few host threads while
 * the previous chunk is on the wire; memory from apo_host_alloc (page-locked) is read in place and
 * reaches PCIe line rate — the binding can hand such memory to JS as an external ArrayBuffer
 * (napi_create_external_arraybuffer, finalizer = apo_host_free). */
int apo_host_alloc(uint64_t bytes, void **out);
int apo_host_free(void *p);
int apo_last_timing(const apo_engine *e, apo_timing *out);
/* Exact partial sums of the last apo_score: per candidate the integer
 * sum_t rint(finalReward * 2^52) as three int64 limbs (value = l2*2^64 + l1*2^32 + l0)
 * and the count; 4*C int64 words.  Order-independent, hence identical for any grid,
 * shard or rank count. */
int apo_debug_partials(apo_engine *e, int64_t *out, uint32_t C);
/* The exception list of the Form T copy (see apo_dims_upload), for tests and diagnostics: *n_exceptions pairs {position in
 * the row, full index} of the evaluations whose index is >= 2^16, rows in order, sorted by position (xs, 2 words each), and
 * its block index (xb, *n_words = C * (blocks per row + 1) words: the list offset of row c's first exception at or after
 * position 8192 b is xb[c * (blocks per row + 1) + b]).  Both counts are 0 when no list is held.  xb / xs may be NULL. */
int apo_debug_twin_t_list(apo_engine *e, uint64_t *n_words, uint64_t *n_exceptions, uint32_t *xb, uint32_t *xs);

/* ---- per-candidate breakdown: why candidate c scored what it scored ------------------
 * The corpus report (APO:498-625) answered per candidate, over the evaluations of c that the
 * scoring call read (every window of a session, absolute record positions).  Built by a scoring
 * call that sets APO_SCORE_CANDIDATES: apo_score, apo_score_finish (every apo_score_accumulate of
 * the session must set it too) or any apo_score_host*.  Feedback tally of an evaluation: Form R /
 * R16 from the feedback field (1 good, 2 bad, else none, whether or not VALID is set, as the
 * corpus scan counts); Form D / Q / P / T from d0 = user_feedback (TCS:677-679): 1 good, -1 bad,
 * anything else (absent included) none.  dim[i] covers the evaluations with a non-null
 * finalReward in which dimension i is present: sum = exact integer sum of rint(v * 2^52) rounded
 * once to binary64 (v = the fp32 value widened for Form D / Q / P / T, the TCS:668-763 binary64
 * value for Form R / R16), avg = sum / count and the flags of APO:575/591/802/819, by the code
 * that fills apo_corpus_report.dim.  A Form R candidate row therefore has the breakdown that the
 * corpus report of that row has on every shared field.  Domain: rint(v * 2^52) is an int64 only
 * for |v| < 2048, so a flagged call fails with APO_E_ARG (and leaves no breakdown) when an
 * evaluation with a non-null finalReward has a present dimension with |v| >= 2048, even where a
 * weight of 0 or cancelling weighted terms keep its finalReward in range; absent values and null
 * evaluations may hold any value.  Single rank only: APO_E_STATE on a handle
 * after apo_comm_init with more than one rank (apo_comm_init with nranks == 1 leaves the handle
 * single-rank, with no communicator, so the breakdown stays available). */
typedef struct apo_candidate_report {
	uint64_t total, good, bad, none;   /* evaluations of c in the scored window(s); tallies as APO:509-516 */
	double   goodRate;                 /* good / (good + bad), 0 when both are 0 (APO:546-547) */
	uint64_t withReward;               /* == counts[c] */
	double   rewardSum, avgReward;     /* avgReward == scores[c] bit for bit; NaN (not -inf) when withReward == 0 */
	apo_dimstat dim[APO_NDIM];         /* same rules and rounding as apo_corpus_report.dim */
	int64_t  badExamples[3];           /* first 3 record indices (ascending) whose tally is 'bad'; -1 = none */
} apo_candidate_report;
/* Breakdown of candidates [c0, c0 + n) from the last scoring call.  APO_E_STATE when that call did
 * not set APO_SCORE_CANDIDATES (or failed), APO_E_ARG when the range exceeds its C. */
int apo_candidate_reports(apo_engine *e, uint32_t c0, uint32_t n, apo_candidate_report *out);
/* Per-candidate corpus report (record sources only): the whole apo_corpus_report of each candidate's scored rollout records.
 * Built by a scoring call that sets APO_SCORE_CANDIDATE_CORPUS (independent of APO_SCORE_CANDIDATES; either or both may be
 * set): apo_score with source APO_SRC_ROLLOUTS (Form R or R16), apo_score_finish (every apo_score_accumulate of the session
 * must set it too) and apo_score_host_records (32- and 16-byte rows).  out[c] is byte for byte the report that apo_score with
 * APO_SCORE_CORPUS produces when candidate c's scored records are the corpus: tallies, goodRate, byMode / byModeGoodRate,
 * withReward / rewardSum / avgReward, dim[9] with its flags, pat[6] with count, flag, severity and examples (no pattern
 * counts when no record is 'bad', APO:641), tool totals and toolSuccessRate.  Example indices are absolute record positions
 * (they include the window's first); a session covers the union of its windows.  Form D / Q / P / T carry none of the record
 * fields the patterns read: APO_E_ARG on those sources and on apo_score_host, apo_score_host_compact, apo_score_host_packed
 * and apo_score_host_tuples.  Single rank only, as the breakdown (APO_E_STATE on a handle with more than one rank).
 * Reports of candidates [c0, c0 + n) of the last scoring call: APO_E_STATE when that call did not set the flag (or failed),
 * APO_E_ARG when the range exceeds its C. */
int apo_candidate_corpus_reports(apo_engine *e, uint32_t c0, uint32_t n, apo_corpus_report *out);

/* ---- multi-GPU: the record axis is sharded across ranks (one process per GPU, or one handle per GPU inside one
 * process); the packed int64 partial vectors of the shards are joined INSIDE the scoring launch: the finalising CTA
 * of every rank publishes its vector in a peer-mapped block, signals the other ranks and sums their vectors with
 * NVLink loads (csrc/apo_corpus.cuh peer_join), so a sharded apo_score is still one kernel launch.  NCCL bootstraps
 * the exchange of the peer handles and remains the fallback (ncclAllReduce(sum,int64) + a finalise launch) when
 * peer memory is unavailable (ranks on different boxes, IPC disabled) or APO_TUNE_NCCL_JOIN is set.  Every joined
 * call (apo_score, apo_score_finish, apo_score_host*) must be made by all ranks in the same order; a rank that never
 * arrives makes the others fail with APO_E_NCCL after 20 s instead of hanging. */
#define APO_UNIQUE_ID_BYTES 128
int apo_comm_unique_id(uint8_t out[APO_UNIQUE_ID_BYTES]);
int apo_comm_init(apo_engine *e, int nranks, int rank, const uint8_t id[APO_UNIQUE_ID_BYTES]);
int apo_comm_destroy(apo_engine *e);
/* 0 = single rank, 1 = ncclAllReduce join, 2 = peer-memory join inside the scoring launch */
int apo_comm_join_mode(const apo_engine *e);

#ifdef __cplusplus
}
#endif
#endif
