/*
 * apo_napi.c — N-API addon over the C ABI of include/apo_b200.h (marshalling only; the job structs, their
 * validation and the per-handle FIFO live in apo_jobs.c so that they are testable without Node).
 *
 * Loaded by the IDE's *main process* (the renderer cannot load native modules: eslint.config.js:94 — `common`
 * imports nothing platform specific), behind a named IPC channel exactly like the reference's metrics service
 * (common/metricsService.ts:25-50 + electron-main/metricsMainService.ts:35, registered in
 * src/vs/code/electron-main/app.ts:1124,1259-1260).  See INTEGRATION.md and ts/.
 *
 * Rules every exported function follows (SURVEY 8b):
 *   - never throws: failures come back as null (create) or a rejected Promise whose Error carries the library's
 *     message (reference convention TCS:438, APO:1211-1214);
 *   - everything that touches the GPU is async work on the libuv pool resolving a Promise ("anything transmitted
 *     over a channel must be async", metricsService.ts:47): the Electron main loop never blocks, not even for the
 *     ~15 us single-trace call;
 *   - one in-flight call per handle: jobs of a handle run strictly in submission order (ticket FIFO, apo_jobs.h);
 *   - ownership: every ArrayBuffer a job reads and the handle itself stay napi_ref'd until the job completed, so
 *     neither the data nor the engine can be collected under a running job; nothing is retained afterwards;
 *   - every shape that arrives over IPC (C, T, K, rowBytes, byte lengths) is validated against the real buffer
 *     lengths with overflow-safe arithmetic before a pointer is dereferenced (apo_job_validate).
 *
 * JS surface:
 *   create(device) -> handle | null        lastCreateError() -> string
 *   dimsUpload(h, dims:ArrayBuffer f32[C][T][9], C, T, compact:boolean)      -> Promise<void>     uploaded once ...
 *   rolloutsUpload(h, recs:ArrayBuffer, rowBytes 32|16, C, T)               -> Promise<void>
 *   corpusUpload(h, recs:ArrayBuffer apo_record[T], idxBase)                -> Promise<void>
 *   corpusUploadJson(h, utf8:ArrayBuffer, idxBase)                          -> Promise<number>   (records)
 *   dimsTuples(h, cap?)                                                     -> Promise<number>   (nTuples) resident Form T from the loaded dims
 *   recordGroupsUpload(h, labels:ArrayBuffer u8[T], G)                      -> Promise<void>     the record group of every position
 *   candidateRefsUpload(h, refs:ArrayBuffer u32[C])                          -> Promise<void>     the reference of every candidate
 *   scoreResident(h, {C, K, source, corpus, first, count, candidates, candidateCorpus, candidateExtremes, candidateGroups, candidateSpread, candidatePairs, candidateGroupPairs}) -> Promise<blocks>   ... scored many times
 *   score(h, dims, C, T, corpus|null, K, candidates?, candidateExtremes?, candidateGroups?, candidateSpread?, candidatePairs?, candidateGroupPairs?) -> Promise<blocks>   host streaming, Form D
 *   scoreHostRecords(h, recs, rowBytes, C, T, corpus|null, K, candidates?, candidateCorpus?, candidateExtremes?, candidateGroups?, candidateSpread?, candidatePairs?, candidateGroupPairs?) -> Promise<blocks>   host streaming, trace records
 *   scoreHostTuples(h, {tl, th, ...}, C, T, corpus|null, K, candidates?, candidateExtremes?, candidateGroups?, candidateSpread?, candidatePairs?, candidateGroupPairs?) -> Promise<blocks>   host streaming, Form T
 *   candidateGroups is the G the labels were uploaded with (0 / absent: no group scores); so is candidateGroupPairs (0 / absent:
 *   no paired comparisons per record group); a call that names both names one G
 *   rewardBatch(h, recs:ArrayBuffer apo_record[n])                          -> Promise<{dims,masks,finals}>
 *   commUniqueId() -> ArrayBuffer(128) | null     commInit(h, nranks, rank, id) -> Promise<void>
 *   recordsFromJson(utf8) -> ArrayBuffer | null   allocPinned(bytes) -> ArrayBuffer | null      (host-only helpers)
 *   blocks = {scores:ArrayBuffer f64[C], counts:ArrayBuffer u64[C], topk:ArrayBuffer i32[K], report:ArrayBuffer,
 *             candidates?:ArrayBuffer apo_candidate_report[C] (only when the call asked for the per-candidate breakdown),
 *             candidateCorpus?:ArrayBuffer apo_corpus_report[C] (only when a call over rollout records asked for the per-candidate
 *             corpus reports),
 *             candidateExtremes?:ArrayBuffer struct apo_candidate_extremes[C] (only when the call asked for the per-candidate
 *             extremes),
 *             candidateGroups?:ArrayBuffer apo_group_score[C][G] (only when the call asked for the per-candidate group scores),
 *             candidateSpread?:ArrayBuffer struct apo_candidate_spread[C] (only when the call asked for the per-candidate reward
 *             spreads),
 *             candidatePairs?:ArrayBuffer struct apo_candidate_pair[C] (only when the call asked for the paired comparisons),
 *             candidateGroupPairs?:ArrayBuffer struct apo_candidate_pair[C][G] (only when the call asked for the paired comparisons
 *             per record group)}
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "apo_b200.h"
#include "apo_jobs.h"

#if defined(__has_include)
#if __has_include(<node_api.h>)
#include <node_api.h>
#define APO_HAVE_NODE_API 1
#endif
#endif
#ifndef APO_HAVE_NODE_API
#include "node_api_stub.h"
#endif

static char g_create_error[256];

/* ------------------------------------------------------------------------------------------ helpers */
static void serial_finalize(napi_env env, void *data, void *hint) { (void)env; (void)hint; apo_serial_destroy((apo_serial *)data); }

static apo_serial *get_serial(napi_env env, napi_value v)
{
	napi_valuetype t;
	void *p = NULL;
	if (napi_typeof(env, v, &t) != napi_ok || t != napi_external) return NULL;
	if (napi_get_value_external(env, v, &p) != napi_ok) return NULL;
	return (apo_serial *)p;
}

static int get_buffer(napi_env env, napi_value v, const void **p, uint64_t *bytes)
{
	bool is = false;
	void *data = NULL; size_t n = 0;
	if (napi_is_arraybuffer(env, v, &is) != napi_ok || !is) return 0;
	if (napi_get_arraybuffer_info(env, v, &data, &n) != napi_ok) return 0;
	*p = data; *bytes = (uint64_t)n;
	return 1;
}

static int get_u32(napi_env env, napi_value v, uint32_t *out)
{
	napi_valuetype t; double d = 0;
	if (napi_typeof(env, v, &t) != napi_ok || t != napi_number) return 0;
	if (napi_get_value_double(env, v, &d) != napi_ok || !(d >= 0) || d > 4294967295.0 || d != (double)(uint32_t)d) return 0;
	*out = (uint32_t)d;
	return 1;
}

static int get_u64(napi_env env, napi_value v, uint64_t *out)        /* JS numbers: exact integers up to 2^53 */
{
	napi_valuetype t; double d = 0;
	if (napi_typeof(env, v, &t) != napi_ok || t != napi_number) return 0;
	if (napi_get_value_double(env, v, &d) != napi_ok || !(d >= 0) || d > 9007199254740992.0 || d != (double)(uint64_t)d) return 0;
	*out = (uint64_t)d;
	return 1;
}

static int is_nullish(napi_env env, napi_value v)
{
	napi_valuetype t;
	return napi_typeof(env, v, &t) != napi_ok || t == napi_null || t == napi_undefined;
}

static napi_value copy_out(napi_env env, const void *src, size_t bytes)
{
	void *p = NULL; napi_value v = NULL;
	if (napi_create_arraybuffer(env, bytes, &p, &v) != napi_ok) return NULL;
	if (bytes) memcpy(p, src, bytes);
	return v;
}

/* ------------------------------------------------------------------------------------------ async plumbing */
typedef struct {
	apo_serial *s;
	apo_job job;
	napi_deferred deferred;
	napi_async_work work;
	napi_ref keep[9];            /* handle, data buffer, corpus buffer (+ the six arrays of a Form T call) */
	int nkeep;
} call_t;

static void call_execute(napi_env env, void *data)
{
	(void)env;
	call_t *c = (call_t *)data;
	apo_job_run(c->s, &c->job);                     /* waits for its turn on the handle (FIFO), then runs */
}

static napi_value blocks_of(napi_env env, const apo_job *j)
{
	napi_value out = NULL, v;
	const uint32_t C = j->C, K = j->K < j->C ? j->K : j->C;
	napi_create_object(env, &out);
	if ((v = copy_out(env, j->scores, 8u * (size_t)C))) napi_set_named_property(env, out, "scores", v);
	if ((v = copy_out(env, j->counts, 8u * (size_t)C))) napi_set_named_property(env, out, "counts", v);
	if ((v = copy_out(env, j->topk, 4u * (size_t)K))) napi_set_named_property(env, out, "topk", v);
	if ((v = copy_out(env, &j->report, sizeof j->report))) napi_set_named_property(env, out, "report", v);
	if (j->candidates && (v = copy_out(env, j->candidates, sizeof(apo_candidate_report) * (size_t)C))) napi_set_named_property(env, out, "candidates", v);
	if (j->candidate_corpus && (v = copy_out(env, j->candidate_corpus, sizeof(apo_corpus_report) * (size_t)C)))
		napi_set_named_property(env, out, "candidateCorpus", v);
	if (j->candidate_extremes && (v = copy_out(env, j->candidate_extremes, sizeof(struct apo_candidate_extremes) * (size_t)C)))
		napi_set_named_property(env, out, "candidateExtremes", v);
	if (j->candidate_groups && (v = copy_out(env, j->candidate_groups, sizeof(apo_group_score) * (size_t)C * j->G)))
		napi_set_named_property(env, out, "candidateGroups", v);
	if (j->candidate_spread && (v = copy_out(env, j->candidate_spread, sizeof(struct apo_candidate_spread) * (size_t)C)))
		napi_set_named_property(env, out, "candidateSpread", v);
	if (j->candidate_pairs && (v = copy_out(env, j->candidate_pairs, sizeof(struct apo_candidate_pair) * (size_t)C)))
		napi_set_named_property(env, out, "candidatePairs", v);
	if (j->candidate_group_pairs && (v = copy_out(env, j->candidate_group_pairs, sizeof(struct apo_candidate_pair) * (size_t)C * j->G)))
		napi_set_named_property(env, out, "candidateGroupPairs", v);
	return out;
}

static void call_complete(napi_env env, napi_status st, void *data)
{
	(void)st;
	call_t *c = (call_t *)data;
	apo_job *j = &c->job;
	if (j->rc != APO_OK) {
		napi_value msg, err;
		napi_create_string_utf8(env, j->err[0] ? j->err : "apo_b200 call failed", NAPI_AUTO_LENGTH, &msg);
		napi_create_error(env, NULL, msg, &err);
		napi_reject_deferred(env, c->deferred, err);
	} else {
		napi_value out = NULL, v;
		switch (j->kind) {
		case APO_JOB_SCORE_RESIDENT: case APO_JOB_SCORE_HOST: case APO_JOB_SCORE_HOST_RECORDS: case APO_JOB_SCORE_HOST_TUPLES:
			out = blocks_of(env, j);
			break;
		case APO_JOB_REWARD_BATCH:
			napi_create_object(env, &out);
			if ((v = copy_out(env, j->dims_out, 8u * APO_NDIM * (size_t)j->n_out))) napi_set_named_property(env, out, "dims", v);
			if ((v = copy_out(env, j->masks_out, 4u * (size_t)j->n_out))) napi_set_named_property(env, out, "masks", v);
			if ((v = copy_out(env, j->finals_out, 8u * (size_t)j->n_out))) napi_set_named_property(env, out, "finals", v);
			break;
		case APO_JOB_CORPUS_UPLOAD_JSON: case APO_JOB_DIMS_TUPLES:
			napi_create_double(env, (double)j->n_out, &out);
			break;
		default:
			napi_get_null(env, &out);
		}
		napi_resolve_deferred(env, c->deferred, out);
	}
	for (int i = 0; i < c->nkeep; i++) napi_delete_reference(env, c->keep[i]);
	napi_delete_async_work(env, c->work);
	apo_job_release(j);
	free(c);
}

/* Validates, takes the handle's ticket and queues the job.  A job that fails validation is still queued (it rejects in
 * its turn): tickets stay dense and the Promise order seen by JS matches the submission order. */
static napi_value submit(napi_env env, call_t *c, napi_value handle, napi_value buf, napi_value corpus, const char *name)
{
	napi_value promise = NULL, rname;
	napi_create_promise(env, &c->deferred, &promise);
	if (apo_job_validate(&c->job) == APO_OK) apo_job_prepare(&c->job);
	c->job.ticket = apo_serial_ticket(c->s);
	napi_create_reference(env, handle, 1, &c->keep[c->nkeep++]);            /* the engine cannot be finalized under the job */
	if (buf) napi_create_reference(env, buf, 1, &c->keep[c->nkeep++]);
	if (corpus) napi_create_reference(env, corpus, 1, &c->keep[c->nkeep++]);
	napi_create_string_utf8(env, name, NAPI_AUTO_LENGTH, &rname);
	napi_create_async_work(env, NULL, rname, call_execute, call_complete, c, &c->work);
	napi_queue_async_work(env, c->work);
	return promise;
}

/* a Promise rejected on the spot: the handle itself is unusable, so there is no FIFO to take a turn in */
static napi_value reject_now(napi_env env, const char *why)
{
	napi_deferred d; napi_value promise = NULL, msg, err;
	napi_create_promise(env, &d, &promise);
	napi_create_string_utf8(env, why, NAPI_AUTO_LENGTH, &msg);
	napi_create_error(env, NULL, msg, &err);
	napi_reject_deferred(env, d, err);
	return promise;
}

static call_t *new_call(napi_env env, napi_value handle, apo_job_kind kind)
{
	apo_serial *s = get_serial(env, handle);
	if (!s) return NULL;
	call_t *c = (call_t *)calloc(1, sizeof *c);
	if (!c) return NULL;
	c->s = s; c->job.kind = kind;
	return c;
}

static void arg_error(call_t *c, const char *msg) { c->job.rc = APO_E_ARG; snprintf(c->job.err, sizeof c->job.err, "%s", msg); }

#define ARGS(n)                                                    \
	size_t argc = (n); napi_value argv[(n)];                       \
	for (size_t i_ = 0; i_ < (n); i_++) argv[i_] = NULL;           \
	napi_get_cb_info(env, info, &argc, argv, NULL, NULL);

/* ------------------------------------------------------------------------------------------ exported functions */
/* create(device:number) -> external handle, or null (lastCreateError() tells why): never throws */
static napi_value Create(napi_env env, napi_callback_info info)
{
	ARGS(1)
	int32_t dev = 0;
	napi_value out = NULL;
	if (argc > 0 && argv[0]) napi_get_value_int32(env, argv[0], &dev);
	apo_serial *s = apo_serial_create(dev, g_create_error, sizeof g_create_error);
	if (!s) { napi_get_null(env, &out); return out; }
	if (napi_create_external(env, s, serial_finalize, NULL, &out) != napi_ok) { apo_serial_destroy(s); napi_get_null(env, &out); }
	return out;
}

static napi_value LastCreateError(napi_env env, napi_callback_info info)
{
	(void)info;
	napi_value out = NULL;
	napi_create_string_utf8(env, g_create_error, NAPI_AUTO_LENGTH, &out);
	return out;
}

/* dimsUpload(h, dims, C, T, compact) */
static napi_value DimsUpload(napi_env env, napi_callback_info info)
{
	ARGS(5)
	call_t *c = argc >= 1 ? new_call(env, argv[0], APO_JOB_DIMS_UPLOAD) : NULL;
	if (!c) return reject_now(env, "dimsUpload: invalid handle");
	bool compact = false;
	if (argc < 4 || !get_buffer(env, argv[1], &c->job.buf, &c->job.buf_bytes) || !get_u32(env, argv[2], &c->job.C) || !get_u64(env, argv[3], &c->job.T))
		arg_error(c, "dimsUpload(handle, dims:ArrayBuffer, C:uint32, T:uint53, compact?:boolean)");
	if (argc >= 5 && argv[4] && !is_nullish(env, argv[4])) napi_get_value_bool(env, argv[4], &compact);
	c->job.compact = compact ? 1 : 0;
	return submit(env, c, argv[0], c->job.buf ? argv[1] : NULL, NULL, "apo_dims_upload");
}

/* rolloutsUpload(h, recs, rowBytes, C, T) */
static napi_value RolloutsUpload(napi_env env, napi_callback_info info)
{
	ARGS(5)
	call_t *c = argc >= 1 ? new_call(env, argv[0], APO_JOB_ROLLOUTS_UPLOAD) : NULL;
	if (!c) return reject_now(env, "rolloutsUpload: invalid handle");
	if (argc < 5 || !get_buffer(env, argv[1], &c->job.buf, &c->job.buf_bytes) || !get_u32(env, argv[2], &c->job.row_bytes) ||
	    !get_u32(env, argv[3], &c->job.C) || !get_u64(env, argv[4], &c->job.T))
		arg_error(c, "rolloutsUpload(handle, recs:ArrayBuffer, rowBytes:32|16, C:uint32, T:uint53)");
	return submit(env, c, argv[0], c->job.buf ? argv[1] : NULL, NULL, "apo_rollouts_upload");
}

/* corpusUpload(h, recs, idxBase) */
static napi_value CorpusUpload(napi_env env, napi_callback_info info)
{
	ARGS(3)
	call_t *c = argc >= 1 ? new_call(env, argv[0], APO_JOB_CORPUS_UPLOAD) : NULL;
	if (!c) return reject_now(env, "corpusUpload: invalid handle");
	if (argc < 2 || !get_buffer(env, argv[1], &c->job.buf, &c->job.buf_bytes)) arg_error(c, "corpusUpload(handle, recs:ArrayBuffer, idxBase?:uint53)");
	if (argc >= 3 && argv[2] && !is_nullish(env, argv[2]) && !get_u64(env, argv[2], &c->job.idx_base)) arg_error(c, "corpusUpload: idxBase must be a non-negative integer");
	return submit(env, c, argv[0], c->job.buf ? argv[1] : NULL, NULL, "apo_corpus_upload");
}

/* corpusUploadJson(h, utf8, idxBase) -> Promise<number of records> */
static napi_value CorpusUploadJson(napi_env env, napi_callback_info info)
{
	ARGS(3)
	call_t *c = argc >= 1 ? new_call(env, argv[0], APO_JOB_CORPUS_UPLOAD_JSON) : NULL;
	if (!c) return reject_now(env, "corpusUploadJson: invalid handle");
	if (argc < 2 || !get_buffer(env, argv[1], &c->job.buf, &c->job.buf_bytes)) arg_error(c, "corpusUploadJson(handle, utf8:ArrayBuffer, idxBase?:uint53)");
	if (argc >= 3 && argv[2] && !is_nullish(env, argv[2]) && !get_u64(env, argv[2], &c->job.idx_base)) arg_error(c, "corpusUploadJson: idxBase must be a non-negative integer");
	return submit(env, c, argv[0], c->job.buf ? argv[1] : NULL, NULL, "apo_corpus_upload_json");
}

/* dimsTuples(h, cap?) -> Promise<number of dictionary entries>: apo_dims_tuples, cap defaults to APO_TUPLES_MAX */
static napi_value DimsTuples(napi_env env, napi_callback_info info)
{
	ARGS(2)
	call_t *c = argc >= 1 ? new_call(env, argv[0], APO_JOB_DIMS_TUPLES) : NULL;
	if (!c) return reject_now(env, "dimsTuples: invalid handle");
	c->job.cap = APO_TUPLES_MAX;
	if (argc >= 2 && argv[1] && !is_nullish(env, argv[1]) && !get_u32(env, argv[1], &c->job.cap))
		arg_error(c, "dimsTuples(handle, cap?:uint32 <= 16777215)");
	return submit(env, c, argv[0], NULL, NULL, "apo_dims_tuples");
}

/* recordGroupsUpload(h, labels, G): apo_record_groups_upload; an empty labels buffer releases them */
static napi_value RecordGroupsUpload(napi_env env, napi_callback_info info)
{
	ARGS(3)
	call_t *c = argc >= 1 ? new_call(env, argv[0], APO_JOB_RECORD_GROUPS_UPLOAD) : NULL;
	if (!c) return reject_now(env, "recordGroupsUpload: invalid handle");
	if (argc < 3 || !get_buffer(env, argv[1], &c->job.buf, &c->job.buf_bytes) || !get_u32(env, argv[2], &c->job.G))
		arg_error(c, "recordGroupsUpload(handle, labels:ArrayBuffer, G:uint32 1..64)");
	return submit(env, c, argv[0], c->job.buf ? argv[1] : NULL, NULL, "apo_record_groups_upload");
}

/* candidateRefsUpload(h, refs): apo_candidate_refs_upload with C = refs.byteLength / 4; an empty buffer releases them */
static napi_value CandidateRefsUpload(napi_env env, napi_callback_info info)
{
	ARGS(2)
	call_t *c = argc >= 1 ? new_call(env, argv[0], APO_JOB_CANDIDATE_REFS_UPLOAD) : NULL;
	if (!c) return reject_now(env, "candidateRefsUpload: invalid handle");
	if (argc < 2 || !get_buffer(env, argv[1], &c->job.buf, &c->job.buf_bytes) || c->job.buf_bytes % 4 || c->job.buf_bytes / 4 > 0xFFFFFFFFull)
		arg_error(c, "candidateRefsUpload(handle, refs:ArrayBuffer u32[C])");
	else
		c->job.C = (uint32_t)(c->job.buf_bytes / 4);
	return submit(env, c, argv[0], c->job.buf ? argv[1] : NULL, NULL, "apo_candidate_refs_upload");
}

static int opt_u32(napi_env env, napi_value obj, const char *key, uint32_t *out)
{
	bool has = false; napi_value v;
	if (napi_has_named_property(env, obj, key, &has) != napi_ok || !has) return 1;
	if (napi_get_named_property(env, obj, key, &v) != napi_ok || is_nullish(env, v)) return 1;
	return get_u32(env, v, out);
}
static int opt_u64(napi_env env, napi_value obj, const char *key, uint64_t *out)
{
	bool has = false; napi_value v;
	if (napi_has_named_property(env, obj, key, &has) != napi_ok || !has) return 1;
	if (napi_get_named_property(env, obj, key, &v) != napi_ok || is_nullish(env, v)) return 1;
	return get_u64(env, v, out);
}

/* optional trailing boolean (undefined / null = false) */
static int opt_bool_arg(napi_env env, napi_value v, int *out)
{
	napi_valuetype t; bool b = false;
	*out = 0;
	if (!v || is_nullish(env, v)) return 1;
	if (napi_typeof(env, v, &t) != napi_ok || t != napi_boolean || napi_get_value_bool(env, v, &b) != napi_ok) return 0;
	*out = b ? 1 : 0;
	return 1;
}

/* candidateGroups (g) and candidateGroupPairs (gp) both name the G the labels were uploaded with, and the job holds one G:
 * 0 when a call names a different G for each, else the one it names (0: neither) */
static uint32_t one_G(uint32_t g, uint32_t gp) { return g && gp && g != gp ? 0u : g ? g : gp; }

/* scoreResident(h, {C, K, source?, corpus?, first?, count?, candidates?, candidateCorpus?, candidateExtremes?, candidateGroups?,
 * candidateSpread?, candidatePairs?, candidateGroupPairs?}): scores what dimsUpload / rolloutsUpload / corpusUpload left
 * resident — "uploaded once, scored many times" (SURVEY 8b ownership row); nothing crosses PCIe but the result block. */
static napi_value ScoreResident(napi_env env, napi_callback_info info)
{
	ARGS(2)
	call_t *c = argc >= 1 ? new_call(env, argv[0], APO_JOB_SCORE_RESIDENT) : NULL;
	if (!c) return reject_now(env, "scoreResident: invalid handle");
	napi_valuetype t;
	uint32_t corpus = 0, cands = 0, ccorp = 0, cext = 0, cspr = 0, cpair = 0, g = 0, gp = 0;
	if (argc < 2 || napi_typeof(env, argv[1], &t) != napi_ok || t != napi_object || !opt_u32(env, argv[1], "candidateGroups", &g) ||
	    !opt_u32(env, argv[1], "candidateGroupPairs", &gp) || ((g || gp) && !one_G(g, gp)) ||
	    !opt_u32(env, argv[1], "C", &c->job.C) || !opt_u32(env, argv[1], "K", &c->job.K) || !opt_u32(env, argv[1], "source", &c->job.source) ||
	    !opt_u32(env, argv[1], "corpus", &corpus) || !opt_u64(env, argv[1], "first", &c->job.first) || !opt_u64(env, argv[1], "count", &c->job.count) ||
	    !opt_u32(env, argv[1], "candidates", &cands) || cands > 1 || !opt_u32(env, argv[1], "candidateCorpus", &ccorp) || ccorp > 1 ||
	    !opt_u32(env, argv[1], "candidateExtremes", &cext) || cext > 1 || !opt_u32(env, argv[1], "candidateSpread", &cspr) || cspr > 1 ||
	    !opt_u32(env, argv[1], "candidatePairs", &cpair) || cpair > 1)
		arg_error(c, "scoreResident(handle, {C:uint32, K:uint32, source?:0|1|2, corpus?:0|1, first?:uint53, count?:uint53, candidates?:0|1, candidateCorpus?:0|1, candidateExtremes?:0|1, candidateGroups?:G, candidateSpread?:0|1, candidatePairs?:0|1, candidateGroupPairs?:G (the same G as candidateGroups)})");
	c->job.G = one_G(g, gp);
	if (c->job.C == 0) arg_error(c, "scoreResident: C (the number of uploaded candidates) is required");
	if (c->job.K > c->job.C) arg_error(c, "scoreResident: K exceeds C");
	c->job.flags = (corpus ? APO_SCORE_CORPUS : 0) | (cands ? APO_SCORE_CANDIDATES : 0) | (ccorp ? APO_SCORE_CANDIDATE_CORPUS : 0) |
	               (cext ? APO_SCORE_CANDIDATE_EXTREMES : 0) | (g ? APO_SCORE_CANDIDATE_GROUPS : 0) | (cspr ? APO_SCORE_CANDIDATE_SPREAD : 0) |
	               (cpair ? APO_SCORE_CANDIDATE_PAIRS : 0) | (gp ? APO_SCORE_CANDIDATE_GROUP_PAIRS : 0);
	return submit(env, c, argv[0], NULL, NULL, "apo_score");
}

static napi_value score_host_common(napi_env env, napi_callback_info info, apo_job_kind kind)
{
	const int rec = kind == APO_JOB_SCORE_HOST_RECORDS;
	ARGS(14)
	call_t *c = argc >= 1 ? new_call(env, argv[0], kind) : NULL;
	if (!c) return reject_now(env, "score: invalid handle");
	int cands = 0, ccorp = 0, cext = 0, cspr = 0, cpair = 0;
	uint32_t g = 0, gp = 0;
	const size_t base = rec ? 3 : 2;              /* index of C */
	const size_t need = base + 4;                 /* ..., C, T, corpus, K */
	int ok = argc >= need && get_buffer(env, argv[1], &c->job.buf, &c->job.buf_bytes);
	if (ok && rec) ok = get_u32(env, argv[2], &c->job.row_bytes);
	if (ok) ok = get_u32(env, argv[base], &c->job.C) && get_u64(env, argv[base + 1], &c->job.T) && get_u32(env, argv[base + 3], &c->job.K);
	napi_value corpus = NULL;
	if (ok && !is_nullish(env, argv[base + 2])) {
		ok = get_buffer(env, argv[base + 2], &c->job.corpus, &c->job.corpus_bytes);
		corpus = ok ? argv[base + 2] : NULL;
	}
	if (ok && argc > need) ok = opt_bool_arg(env, argv[need], &cands);
	if (ok && rec && argc > need + 1) ok = opt_bool_arg(env, argv[need + 1], &ccorp);     /* trace records only */
	const size_t ext_at = rec ? need + 2 : need + 1;
	if (ok && argc > ext_at) ok = opt_bool_arg(env, argv[ext_at], &cext);
	if (ok && argc > ext_at + 1 && !is_nullish(env, argv[ext_at + 1])) ok = get_u32(env, argv[ext_at + 1], &g);
	if (ok && argc > ext_at + 2) ok = opt_bool_arg(env, argv[ext_at + 2], &cspr);
	if (ok && argc > ext_at + 3) ok = opt_bool_arg(env, argv[ext_at + 3], &cpair);
	if (ok && argc > ext_at + 4 && !is_nullish(env, argv[ext_at + 4])) ok = get_u32(env, argv[ext_at + 4], &gp);   /* the last optional argument */
	if (ok && (g || gp)) ok = one_G(g, gp) != 0;
	c->job.G = one_G(g, gp);
	c->job.flags = (cands ? APO_SCORE_CANDIDATES : 0) | (ccorp ? APO_SCORE_CANDIDATE_CORPUS : 0) | (cext ? APO_SCORE_CANDIDATE_EXTREMES : 0) |
	               (g ? APO_SCORE_CANDIDATE_GROUPS : 0) | (cspr ? APO_SCORE_CANDIDATE_SPREAD : 0) | (cpair ? APO_SCORE_CANDIDATE_PAIRS : 0) |
	               (gp ? APO_SCORE_CANDIDATE_GROUP_PAIRS : 0);
	if (!ok) arg_error(c, rec ? "scoreHostRecords(handle, recs:ArrayBuffer, rowBytes:32|16, C:uint32, T:uint53, corpus:ArrayBuffer|null, K:uint32, candidates?:boolean, candidateCorpus?:boolean, candidateExtremes?:boolean, candidateGroups?:G, candidateSpread?:boolean, candidatePairs?:boolean, candidateGroupPairs?:G)"
	                          : "score(handle, dims:ArrayBuffer, C:uint32, T:uint53, corpus:ArrayBuffer|null, K:uint32, candidates?:boolean, candidateExtremes?:boolean, candidateGroups?:G, candidateSpread?:boolean, candidatePairs?:boolean, candidateGroupPairs?:G)");
	return submit(env, c, argv[0], c->job.buf ? argv[1] : NULL, corpus, rec ? "apo_score_host_records" : "apo_score_host");
}
static napi_value Score(napi_env env, napi_callback_info info) { return score_host_common(env, info, APO_JOB_SCORE_HOST); }
static napi_value ScoreHostRecords(napi_env env, napi_callback_info info) { return score_host_common(env, info, APO_JOB_SCORE_HOST_RECORDS); }

/* encodeTuples(dims:ArrayBuffer f32[C][T][9], C, T, nthreads?) -> Promise<{tl, th, tbookPc, tbookPd, codebook, d2book, nTuples} | null>.
 * Host-side format code (no engine, no GPU, off the JS thread): Form D -> Form P (apo_packed_encode_host) -> Form T
 * (apo_tuple_encode_host), the 3-byte wire format of scoreHostTuples.  Resolves null when the tensor is not categorical enough
 * for Form P / Form T (the caller keeps score()). */
typedef struct {
	napi_deferred deferred; napi_async_work work; napi_ref keep;
	const float *dims; uint32_t C, nthreads, n; uint64_t T; int rc;
	uint16_t *tl; uint8_t *th; uint32_t *tb_pc; uint16_t *tb_pd;
	uint32_t book[8 * 256], d2book[4096];
} enc_t;

static void enc_execute(napi_env env, void *data)
{
	(void)env;
	enc_t *q = (enc_t *)data;
	const uint64_t N = (uint64_t)q->C * q->T, n1 = N ? N : 1;
	const uint32_t cap = N < APO_TUPLES_MAX ? (uint32_t)n1 : APO_TUPLES_MAX;
	uint32_t *pc = (uint32_t *)malloc((size_t)n1 * 4);
	uint16_t *pd = (uint16_t *)malloc((size_t)n1 * 2);
	q->tl = (uint16_t *)malloc((size_t)n1 * 2); q->th = (uint8_t *)malloc((size_t)n1);
	q->tb_pc = (uint32_t *)malloc((size_t)cap * 4); q->tb_pd = (uint16_t *)malloc((size_t)cap * 2);
	q->rc = APO_E_NOMEM;
	if (pc && pd && q->tl && q->th && q->tb_pc && q->tb_pd) {
		q->rc = apo_packed_encode_host(q->dims, q->C, q->T, pc, pd, q->book, q->d2book, (int)q->nthreads);
		if (q->rc == APO_OK) q->rc = apo_tuple_encode_host(pc, pd, q->C, q->T, q->tl, q->th, q->tb_pc, q->tb_pd, cap, &q->n, (int)q->nthreads);
	}
	free(pc); free(pd);
}

static void free_finalize(napi_env env, void *data, void *hint) { (void)env; (void)hint; free(data); }

static void enc_complete(napi_env env, napi_status st, void *data)
{
	(void)st;
	enc_t *q = (enc_t *)data;
	napi_value out = NULL, v;
	napi_get_null(env, &out);
	if (q->rc == APO_OK) {
		const uint64_t N = (uint64_t)q->C * q->T;
		napi_value vtl = NULL, vth = NULL;
		/* the planes are handed to JS without a copy; everything else is small */
		if (napi_create_external_arraybuffer(env, q->tl, (size_t)N * 2, free_finalize, NULL, &vtl) == napi_ok) q->tl = NULL;
		if (napi_create_external_arraybuffer(env, q->th, (size_t)N, free_finalize, NULL, &vth) == napi_ok) q->th = NULL;
		if (vtl && vth) {
			napi_create_object(env, &out);
			napi_set_named_property(env, out, "tl", vtl); napi_set_named_property(env, out, "th", vth);
			if ((v = copy_out(env, q->tb_pc, (size_t)q->n * 4))) napi_set_named_property(env, out, "tbookPc", v);
			if ((v = copy_out(env, q->tb_pd, (size_t)q->n * 2))) napi_set_named_property(env, out, "tbookPd", v);
			if ((v = copy_out(env, q->book, sizeof q->book))) napi_set_named_property(env, out, "codebook", v);
			if ((v = copy_out(env, q->d2book, sizeof q->d2book))) napi_set_named_property(env, out, "d2book", v);
			napi_create_double(env, (double)q->n, &v); napi_set_named_property(env, out, "nTuples", v);
		}
	}
	napi_resolve_deferred(env, q->deferred, out);
	napi_delete_reference(env, q->keep);
	napi_delete_async_work(env, q->work);
	free(q->tl); free(q->th); free(q->tb_pc); free(q->tb_pd);
	free(q);
}

static napi_value EncodeTuples(napi_env env, napi_callback_info info)
{
	ARGS(4)
	const void *dims = NULL; uint64_t bytes = 0, T = 0; uint32_t C = 0, nthreads = 4;
	if (argc < 3 || !get_buffer(env, argv[0], &dims, &bytes) || !get_u32(env, argv[1], &C) || !get_u64(env, argv[2], &T) ||
	    (argc >= 4 && argv[3] && !is_nullish(env, argv[3]) && !get_u32(env, argv[3], &nthreads)))
		return reject_now(env, "encodeTuples(dims:ArrayBuffer, C:uint32, T:uint53, nthreads?:uint32)");
	if (C == 0 || (T && (uint64_t)C > UINT64_MAX / 36 / T) || (uint64_t)C * T * 36 > bytes) return reject_now(env, "encodeTuples: dims buffer is smaller than C*T*36 bytes");
	enc_t *q = (enc_t *)calloc(1, sizeof *q);
	if (!q) return reject_now(env, "encodeTuples: out of host memory");
	q->dims = (const float *)dims; q->C = C; q->T = T; q->nthreads = nthreads ? nthreads : 1;
	napi_value promise = NULL, rname;
	napi_create_promise(env, &q->deferred, &promise);
	napi_create_reference(env, argv[0], 1, &q->keep);                /* the encoder reads the caller's buffer on a worker thread */
	napi_create_string_utf8(env, "apo_tuple_encode_host", NAPI_AUTO_LENGTH, &rname);
	napi_create_async_work(env, NULL, rname, enc_execute, enc_complete, q, &q->work);
	napi_queue_async_work(env, q->work);
	return promise;
}

/* scoreHostTuples(h, {tl, th, tbookPc, tbookPd, codebook, d2book, nTuples}, C, T, corpus|null, K, candidates?, candidateExtremes?, candidateGroups?,
 * candidateSpread?, candidatePairs?, candidateGroupPairs?) -> Promise<blocks>:
 * the evaluations travel as 3-byte dictionary indices (Form T) instead of 36-byte fp32 rows; same integers, same result. */
static napi_value ScoreHostTuples(napi_env env, napi_callback_info info)
{
	static const char *names[6] = {"tl", "th", "tbookPc", "tbookPd", "codebook", "d2book"};
	ARGS(12)
	call_t *c = argc >= 1 ? new_call(env, argv[0], APO_JOB_SCORE_HOST_TUPLES) : NULL;
	if (!c) return reject_now(env, "scoreHostTuples: invalid handle");
	napi_valuetype t;
	napi_value arr[6] = {NULL, NULL, NULL, NULL, NULL, NULL}, corpus = NULL;
	int ok = argc >= 6 && napi_typeof(env, argv[1], &t) == napi_ok && t == napi_object;
	for (int i = 0; ok && i < 6; i++) {
		ok = napi_get_named_property(env, argv[1], names[i], &arr[i]) == napi_ok &&
		     (i == 0 ? get_buffer(env, arr[i], &c->job.buf, &c->job.buf_bytes) : get_buffer(env, arr[i], &c->job.aux[i - 1], &c->job.aux_bytes[i - 1]));
		if (!ok) arr[i] = NULL;
	}
	if (ok) ok = opt_u32(env, argv[1], "nTuples", &c->job.n_tuples) && get_u32(env, argv[2], &c->job.C) && get_u64(env, argv[3], &c->job.T) && get_u32(env, argv[5], &c->job.K);
	if (ok && !is_nullish(env, argv[4])) {
		ok = get_buffer(env, argv[4], &c->job.corpus, &c->job.corpus_bytes);
		corpus = ok ? argv[4] : NULL;
	}
	int cands = 0, cext = 0, cspr = 0, cpair = 0;
	uint32_t g = 0, gp = 0;
	if (ok && argc > 6) ok = opt_bool_arg(env, argv[6], &cands);
	if (ok && argc > 7) ok = opt_bool_arg(env, argv[7], &cext);
	if (ok && argc > 8 && !is_nullish(env, argv[8])) ok = get_u32(env, argv[8], &g);
	if (ok && argc > 9) ok = opt_bool_arg(env, argv[9], &cspr);
	if (ok && argc > 10) ok = opt_bool_arg(env, argv[10], &cpair);
	if (ok && argc > 11 && !is_nullish(env, argv[11])) ok = get_u32(env, argv[11], &gp);
	if (ok && (g || gp)) ok = one_G(g, gp) != 0;
	c->job.G = one_G(g, gp);
	c->job.flags = (cands ? APO_SCORE_CANDIDATES : 0) | (cext ? APO_SCORE_CANDIDATE_EXTREMES : 0) | (g ? APO_SCORE_CANDIDATE_GROUPS : 0) |
	               (cspr ? APO_SCORE_CANDIDATE_SPREAD : 0) | (cpair ? APO_SCORE_CANDIDATE_PAIRS : 0) | (gp ? APO_SCORE_CANDIDATE_GROUP_PAIRS : 0);
	if (!ok) arg_error(c, "scoreHostTuples(handle, {tl, th, tbookPc, tbookPd, codebook, d2book: ArrayBuffer, nTuples:uint32}, C:uint32, T:uint53, corpus:ArrayBuffer|null, K:uint32, candidates?:boolean, candidateExtremes?:boolean, candidateGroups?:G, candidateSpread?:boolean, candidatePairs?:boolean, candidateGroupPairs?:G)");
	for (int i = 1; i < 6; i++)                                      /* the job reads these on a worker thread: keep them alive */
		if (arr[i]) napi_create_reference(env, arr[i], 1, &c->keep[c->nkeep++]);
	return submit(env, c, argv[0], arr[0], corpus, "apo_score_host_tuples");
}

/* rewardBatch(h, recs) -> Promise<{dims, masks, finals}> = TraceCollectorService._computeRewardSignals for n traces
 * (TCS:668-788).  Async like everything else; the TS service micro-batches the single-trace calls of one tick. */
static napi_value RewardBatch(napi_env env, napi_callback_info info)
{
	ARGS(2)
	call_t *c = argc >= 1 ? new_call(env, argv[0], APO_JOB_REWARD_BATCH) : NULL;
	if (!c) return reject_now(env, "rewardBatch: invalid handle");
	if (argc < 2 || !get_buffer(env, argv[1], &c->job.buf, &c->job.buf_bytes)) arg_error(c, "rewardBatch(handle, records:ArrayBuffer)");
	return submit(env, c, argv[0], c->job.buf ? argv[1] : NULL, NULL, "apo_reward_batch");
}

/* commUniqueId() -> ArrayBuffer(128) | null;  commInit(h, nranks, rank, id) -> Promise<void> */
static napi_value CommUniqueId(napi_env env, napi_callback_info info)
{
	(void)info;
	uint8_t id[APO_UNIQUE_ID_BYTES];
	napi_value out = NULL;
	if (apo_comm_unique_id(id) != APO_OK) { napi_get_null(env, &out); return out; }
	out = copy_out(env, id, sizeof id);
	if (!out) napi_get_null(env, &out);
	return out;
}

static napi_value CommInit(napi_env env, napi_callback_info info)
{
	ARGS(4)
	call_t *c = argc >= 1 ? new_call(env, argv[0], APO_JOB_COMM_INIT) : NULL;
	if (!c) return reject_now(env, "commInit: invalid handle");
	const void *id = NULL; uint64_t idb = 0; int32_t nr = 0, rk = 0;
	if (argc < 4 || napi_get_value_int32(env, argv[1], &nr) != napi_ok || napi_get_value_int32(env, argv[2], &rk) != napi_ok ||
	    !get_buffer(env, argv[3], &id, &idb) || idb != APO_UNIQUE_ID_BYTES)
		arg_error(c, "commInit(handle, nranks:int, rank:int, id:ArrayBuffer(128))");
	else { c->job.nranks = nr; c->job.rank = rk; memcpy(c->job.comm_id, id, APO_UNIQUE_ID_BYTES); }
	return submit(env, c, argv[0], NULL, NULL, "apo_comm_init");
}

/* allocPinned(bytes) -> ArrayBuffer over page-locked memory (apo_host_alloc) | null.  Typed arrays built on it are read in
 * place by the streaming calls at PCIe line rate; ordinary ArrayBuffers work too (threaded pinned staging, about half). */
static void pinned_finalize(napi_env env, void *data, void *hint) { (void)env; (void)hint; apo_host_free(data); }

static napi_value AllocPinned(napi_env env, napi_callback_info info)
{
	ARGS(1)
	napi_value out = NULL; uint64_t bytes = 0; void *p = NULL;
	if (argc < 1 || !get_u64(env, argv[0], &bytes) || apo_host_alloc(bytes, &p) != APO_OK) { napi_get_null(env, &out); return out; }
	if (napi_create_external_arraybuffer(env, p, (size_t)bytes, pinned_finalize, NULL, &out) != napi_ok) { apo_host_free(p); napi_get_null(env, &out); }
	return out;
}

/* recordsFromJson(utf8:ArrayBuffer) -> ArrayBuffer of apo_record[T] | null (malformed).  utf8 = the string stored under
 * 'senweaver.traceCollector.data' (TCS:296-359).  Host-side format code, linear in the input, no GPU work. */
static napi_value RecordsFromJson(napi_env env, napi_callback_info info)
{
	ARGS(1)
	napi_value out = NULL;
	const void *text = NULL; uint64_t bytes = 0, pos = 0;
	if (argc < 1 || !get_buffer(env, argv[0], &text, &bytes)) { napi_get_null(env, &out); return out; }
	const int64_t n = apo_records_from_json((const char *)text, bytes, NULL, 0, &pos);
	void *recs = NULL;
	if (n < 0 || napi_create_arraybuffer(env, (size_t)n * sizeof(apo_record), &recs, &out) != napi_ok) { napi_get_null(env, &out); return out; }
	if (n) apo_records_from_json((const char *)text, bytes, (apo_record *)recs, (uint64_t)n, &pos);
	return out;
}

NAPI_MODULE_INIT()
{
	const napi_property_descriptor props[] = {
	    {"create", NULL, Create, NULL, NULL, NULL, napi_default, NULL},
	    {"lastCreateError", NULL, LastCreateError, NULL, NULL, NULL, napi_default, NULL},
	    {"dimsUpload", NULL, DimsUpload, NULL, NULL, NULL, napi_default, NULL},
	    {"rolloutsUpload", NULL, RolloutsUpload, NULL, NULL, NULL, napi_default, NULL},
	    {"corpusUpload", NULL, CorpusUpload, NULL, NULL, NULL, napi_default, NULL},
	    {"corpusUploadJson", NULL, CorpusUploadJson, NULL, NULL, NULL, napi_default, NULL},
	    {"dimsTuples", NULL, DimsTuples, NULL, NULL, NULL, napi_default, NULL},
	    {"recordGroupsUpload", NULL, RecordGroupsUpload, NULL, NULL, NULL, napi_default, NULL},
	    {"candidateRefsUpload", NULL, CandidateRefsUpload, NULL, NULL, NULL, napi_default, NULL},
	    {"scoreResident", NULL, ScoreResident, NULL, NULL, NULL, napi_default, NULL},
	    {"score", NULL, Score, NULL, NULL, NULL, napi_default, NULL},
	    {"scoreHostRecords", NULL, ScoreHostRecords, NULL, NULL, NULL, napi_default, NULL},
	    {"encodeTuples", NULL, EncodeTuples, NULL, NULL, NULL, napi_default, NULL},
	    {"scoreHostTuples", NULL, ScoreHostTuples, NULL, NULL, NULL, napi_default, NULL},
	    {"rewardBatch", NULL, RewardBatch, NULL, NULL, NULL, napi_default, NULL},
	    {"commUniqueId", NULL, CommUniqueId, NULL, NULL, NULL, napi_default, NULL},
	    {"commInit", NULL, CommInit, NULL, NULL, NULL, napi_default, NULL},
	    {"allocPinned", NULL, AllocPinned, NULL, NULL, NULL, napi_default, NULL},
	    {"recordsFromJson", NULL, RecordsFromJson, NULL, NULL, NULL, napi_default, NULL},
	};
	napi_define_properties(env, exports, sizeof props / sizeof props[0], props);
	return exports;
}
