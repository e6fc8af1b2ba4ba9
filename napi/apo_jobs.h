/*
 * apo_jobs.h — the N-API-independent core of the addon (napi/apo_napi.c): one job struct per exported JS call,
 * argument validation, and a per-handle FIFO that honours the C ABI's threading rule ("a handle is not
 * re-entrant: one in-flight call per handle", include/apo_b200.h).
 *
 * The JS thread takes a ticket when it submits a job (apo_serial_ticket — strictly increasing, JS thread only);
 * the libuv worker that executes the job waits until every earlier ticket of the same handle has finished
 * (apo_job_run).  libuv dequeues in submission order, so a job never waits for a ticket that has not been
 * dequeued yet: no deadlock, and jobs of one handle run in exactly the order JS issued them
 * (upload -> score sequences keep their meaning; overlapping score() promises cannot race on the handle).
 *
 * Plain C + pthreads so that tests drive the same structs without Node (tests/c/).
 * Reference conventions kept: never throw into the caller (TCS:438, APO:1211-1214) — every failure is a
 * return code + message; async only across the IPC channel (common/metricsService.ts:47).
 */
#ifndef APO_JOBS_H
#define APO_JOBS_H
#include <pthread.h>
#include <stddef.h>
#include <stdint.h>
#include "apo_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct apo_serial {
	apo_engine *e;                 /* NULL only for the host-only test serials (apo_serial_create_detached) */
	pthread_mutex_t mu;
	pthread_cond_t cv;
	uint64_t next_ticket;          /* JS thread */
	uint64_t serving;              /* ticket allowed to run */
	char create_error[256];
} apo_serial;

/* Never throws / aborts: returns NULL and fills err when no H100 or no library (the TS side logs and disables the fast path). */
apo_serial *apo_serial_create(int device, char *err, size_t errlen);
apo_serial *apo_serial_create_detached(void);          /* no engine: host-format jobs and tests only */
void apo_serial_destroy(apo_serial *s);                /* waits for every issued ticket, then apo_destroy */
uint64_t apo_serial_ticket(apo_serial *s);

typedef enum {
	APO_JOB_DIMS_UPLOAD = 1,       /* dimsUpload(handle, dims f32[C][T][9], C, T, compact)      */
	APO_JOB_ROLLOUTS_UPLOAD,       /* rolloutsUpload(handle, recs, rowBytes 32|16, C, T)         */
	APO_JOB_CORPUS_UPLOAD,         /* corpusUpload(handle, recs apo_record[T], idxBase)          */
	APO_JOB_CORPUS_UPLOAD_JSON,    /* corpusUploadJson(handle, utf8, idxBase)                    */
	APO_JOB_SCORE_RESIDENT,        /* scoreResident(handle, {K, source, corpus, first, count, candidates, candidateCorpus, candidateExtremes, candidateGroups, candidateSpread, candidatePairs, candidateGroupPairs}) */
	APO_JOB_SCORE_HOST,            /* score(handle, dims, C, T, corpus|null, K, candidates?, candidateExtremes?, candidateGroups?, candidateSpread?, candidatePairs?, candidateGroupPairs?) */
	APO_JOB_SCORE_HOST_RECORDS,    /* scoreHostRecords(handle, recs, rowBytes, C, T, corpus|null, K, candidates?, candidateCorpus?, candidateExtremes?, candidateGroups?, candidateSpread?, candidatePairs?, candidateGroupPairs?) */
	APO_JOB_SCORE_HOST_TUPLES,     /* scoreHostTuples(handle, {tl, th, tbookPc, tbookPd, codebook, d2book}, C, T, corpus|null, K, candidates?, candidateExtremes?, candidateGroups?, candidateSpread?, candidatePairs?, candidateGroupPairs?) */
	APO_JOB_REWARD_BATCH,          /* rewardBatch(handle, recs apo_record[n])                    */
	APO_JOB_COMM_INIT,             /* commInit(handle, nranks, rank, id[128])                    */
	APO_JOB_TEST_HOOK,             /* tests: calls hook(hook_arg) in its turn                    */
	APO_JOB_DIMS_TUPLES,           /* dimsTuples(handle, cap?) -> nTuples: resident Form T built from the loaded dims */
	APO_JOB_RECORD_GROUPS_UPLOAD,  /* recordGroupsUpload(handle, labels u8[T], G): the record group of every position */
	APO_JOB_CANDIDATE_REFS_UPLOAD  /* candidateRefsUpload(handle, refs u32[C]): the reference of every candidate (or APO_PAIR_NONE) */
} apo_job_kind;

typedef struct apo_job {
	apo_job_kind kind;
	uint64_t ticket;
	/* inputs (host pointers stay owned and ref'd by the caller until the job completed) */
	const void *buf; uint64_t buf_bytes;          /* dims / records / utf8 */
	const void *corpus; uint64_t corpus_bytes;    /* optional apo_record[Tc] uploaded before a host scoring call */
	const void *aux[5]; uint64_t aux_bytes[5];    /* Form T: th plane, tbook_pc, tbook_pd, codebook (8 x 256 u32), d2book (4096 u32); buf = tl plane */
	uint32_t n_tuples;
	uint32_t cap;                                 /* dimsTuples: dictionary capacity, <= APO_TUPLES_MAX */
	uint32_t C, K, row_bytes, source, flags;
	uint32_t G;                                   /* recordGroupsUpload: groups of the labels; scoring jobs with APO_SCORE_CANDIDATE_GROUPS: the G they were uploaded with */
	uint64_t T, first, count, idx_base;
	int compact;
	int nranks, rank; uint8_t comm_id[APO_UNIQUE_ID_BYTES];
	void (*hook)(void *); void *hook_arg;
	/* outputs (allocated by apo_job_prepare, released by apo_job_release) */
	double *scores; uint64_t *counts; int32_t *topk; apo_corpus_report report;
	apo_candidate_report *candidates;             /* [C], only when flags has APO_SCORE_CANDIDATES (apo_candidate_reports) */
	apo_corpus_report *candidate_corpus;          /* [C], only when flags has APO_SCORE_CANDIDATE_CORPUS (apo_candidate_corpus_reports) */
	struct apo_candidate_extremes *candidate_extremes;   /* [C], only when flags has APO_SCORE_CANDIDATE_EXTREMES (apo_candidate_extremes) */
	apo_group_score *candidate_groups;            /* [C][G], only when flags has APO_SCORE_CANDIDATE_GROUPS (apo_candidate_groups) */
	struct apo_candidate_spread *candidate_spread;   /* [C], only when flags has APO_SCORE_CANDIDATE_SPREAD (apo_candidate_spread) */
	struct apo_candidate_pair *candidate_pairs;      /* [C], only when flags has APO_SCORE_CANDIDATE_PAIRS (apo_candidate_pairs) */
	struct apo_candidate_pair *candidate_group_pairs;   /* [C][G], only when flags has APO_SCORE_CANDIDATE_GROUP_PAIRS (apo_candidate_group_pairs) */
	double *dims_out; uint32_t *masks_out; double *finals_out; uint64_t n_out;
	int rc; char err[256];
} apo_job;

/* Largest per-candidate breakdown a job hands back (one ArrayBuffer of C x sizeof(apo_candidate_report) = 376 B):
 * 4 GiB, about 11.4 M candidates.  Larger requests are refused by apo_job_validate instead of overflowing. */
#define APO_JOB_CANDIDATES_MAX_BYTES (1ull << 32)
/* Same cap for the per-candidate corpus reports (C x sizeof(apo_corpus_report) = 784 B): about 5.5 M candidates.  They exist
 * for record jobs only (scoreResident with source APO_SRC_ROLLOUTS, scoreHostRecords); every other job is refused. */
#define APO_JOB_CANDIDATE_CORPUS_MAX_BYTES (1ull << 32)
/* Same cap for the per-candidate extremes (C x sizeof(struct apo_candidate_extremes) = 1032 B): about 4.16 M candidates.
 * They belong to every scoring job. */
#define APO_JOB_CANDIDATE_EXTREMES_MAX_BYTES (1ull << 32)
/* Same cap for the per-candidate group scores (C x G x sizeof(apo_group_score) = 56 B each).  They belong to every scoring job. */
#define APO_JOB_CANDIDATE_GROUPS_MAX_BYTES (1ull << 32)
/* Same cap for the per-candidate reward spreads (C x sizeof(struct apo_candidate_spread) = 88 B).  They belong to every
 * scoring job. */
#define APO_JOB_CANDIDATE_SPREAD_MAX_BYTES (1ull << 32)
/* Same cap for the paired comparisons (C x sizeof(struct apo_candidate_pair) = 128 B).  They belong to every scoring job. */
#define APO_JOB_CANDIDATE_PAIRS_MAX_BYTES (1ull << 32)
/* Same cap for the paired comparisons per record group (C x G x sizeof(struct apo_candidate_pair) = 128 B each).  They belong
 * to every scoring job and split by the job's G. */
#define APO_JOB_CANDIDATE_GROUP_PAIRS_MAX_BYTES (1ull << 32)

/* Shape / size / overflow checks that need no engine; 0 = fine, else APO_E_ARG with the reason in j->err.
 * Everything that arrives from the renderer over IPC passes through here before a pointer is dereferenced. */
int apo_job_validate(apo_job *j);
/* Allocates the output arrays of the job kind (after validate). */
int apo_job_prepare(apo_job *j);
/* Waits for the job's turn on the handle, runs it through the C ABI, lets the next ticket in.  Worker thread. */
void apo_job_run(apo_serial *s, apo_job *j);
void apo_job_release(apo_job *j);

#ifdef __cplusplus
}
#endif
#endif
