/* apo_jobs.c — see apo_jobs.h.  Everything here is reachable from tests without Node. */
#include "apo_jobs.h"
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

static apo_serial *serial_new(void)
{
	apo_serial *s = (apo_serial *)calloc(1, sizeof *s);
	if (!s) return NULL;
	pthread_mutex_init(&s->mu, NULL);
	pthread_cond_init(&s->cv, NULL);
	return s;
}

apo_serial *apo_serial_create(int device, char *err, size_t errlen)
{
	apo_serial *s = serial_new();
	if (!s) { if (err && errlen) snprintf(err, errlen, "out of host memory"); return NULL; }
	if (apo_create(device, &s->e) != APO_OK) {
		if (err && errlen) snprintf(err, errlen, "%s", apo_last_error(NULL));
		pthread_cond_destroy(&s->cv); pthread_mutex_destroy(&s->mu); free(s);
		return NULL;
	}
	return s;
}

apo_serial *apo_serial_create_detached(void) { return serial_new(); }

uint64_t apo_serial_ticket(apo_serial *s) { return s->next_ticket++; }

void apo_serial_destroy(apo_serial *s)
{
	if (!s) return;
	pthread_mutex_lock(&s->mu);
	while (s->serving < s->next_ticket) pthread_cond_wait(&s->cv, &s->mu);    /* jobs in flight finish first */
	pthread_mutex_unlock(&s->mu);
	if (s->e) apo_destroy(s->e);
	pthread_cond_destroy(&s->cv); pthread_mutex_destroy(&s->mu);
	free(s);
}

static int bad(apo_job *j, const char *msg) { snprintf(j->err, sizeof j->err, "%s", msg); j->rc = APO_E_ARG; return APO_E_ARG; }

/* a * b * c <= limit without overflow */
static int fits(uint64_t a, uint64_t b, uint64_t c, uint64_t limit)
{
	if (a == 0 || b == 0 || c == 0) return 1;
	if (a > limit / b) return 0;
	if (a * b > limit / c) return 0;
	return 1;
}

int apo_job_validate(apo_job *j)
{
	if (j->rc != APO_OK) return j->rc;            /* the marshalling layer already rejected the arguments */
	j->err[0] = 0;
	switch (j->kind) {
	case APO_JOB_DIMS_UPLOAD:
	case APO_JOB_SCORE_HOST:
		if (!j->buf) return bad(j, "dims buffer missing");
		if (j->C == 0) return bad(j, "C must be > 0");
		if (!fits(j->C, j->T, 36, j->buf_bytes)) return bad(j, "dims buffer is smaller than C*T*36 bytes");
		break;
	case APO_JOB_ROLLOUTS_UPLOAD:
	case APO_JOB_SCORE_HOST_RECORDS:
		if (!j->buf) return bad(j, "records buffer missing");
		if (j->C == 0) return bad(j, "C must be > 0");
		if (j->row_bytes != 32 && j->row_bytes != 16) return bad(j, "rowBytes must be 32 or 16");
		if (!fits(j->C, j->T, j->row_bytes, j->buf_bytes)) return bad(j, "records buffer is smaller than C*T*rowBytes");
		break;
	case APO_JOB_SCORE_HOST_TUPLES:
		if (j->C == 0) return bad(j, "C must be > 0");
		if (j->T && (!j->buf || !j->aux[0])) return bad(j, "index planes missing");
		if (!fits(j->C, j->T, 2, j->buf_bytes)) return bad(j, "tl plane is smaller than C*T*2 bytes");
		if (!fits(j->C, j->T, 1, j->aux_bytes[0])) return bad(j, "th plane is smaller than C*T bytes");
		if (j->n_tuples > APO_TUPLES_MAX) return bad(j, "more than 16777215 dictionary entries");
		if (j->T && j->n_tuples == 0) return bad(j, "evaluations without a dictionary");
		if (j->n_tuples && (!j->aux[1] || !j->aux[2])) return bad(j, "dictionary missing");
		if (j->aux_bytes[1] / 4 < j->n_tuples || j->aux_bytes[2] / 2 < j->n_tuples) return bad(j, "dictionary arrays are shorter than nTuples entries");
		if (!j->aux[3] || j->aux_bytes[3] != 8u * 256u * 4u) return bad(j, "codebook must be 8 x 256 uint32");
		if (!j->aux[4] || j->aux_bytes[4] != 4096u * 4u) return bad(j, "d2book must be 4096 uint32");
		break;
	case APO_JOB_CORPUS_UPLOAD:
		if (!j->buf && j->buf_bytes) return bad(j, "corpus buffer missing");
		if (j->buf_bytes % sizeof(apo_record)) return bad(j, "corpus byte length is not a multiple of 32");
		break;
	case APO_JOB_CORPUS_UPLOAD_JSON:
		if (!j->buf) return bad(j, "json buffer missing");
		break;
	case APO_JOB_SCORE_RESIDENT:
		if (j->source > APO_SRC_TUPLES) return bad(j, "unknown source");
		if (j->first % 4) return bad(j, "window start must be a multiple of 4");
		break;
	case APO_JOB_REWARD_BATCH:
		if (!j->buf && j->buf_bytes) return bad(j, "records buffer missing");
		if (j->buf_bytes % sizeof(apo_record)) return bad(j, "records byte length is not a multiple of 32");
		break;
	case APO_JOB_COMM_INIT:
		if (j->nranks < 1 || j->rank < 0 || j->rank >= j->nranks) return bad(j, "bad rank / nranks");
		break;
	case APO_JOB_DIMS_TUPLES:
		if (j->cap > APO_TUPLES_MAX) return bad(j, "cap exceeds 16777215 dictionary entries");
		break;
	case APO_JOB_RECORD_GROUPS_UPLOAD:                /* buf_bytes = T labels; T == 0 releases them */
		if (j->buf_bytes && !j->buf) return bad(j, "labels buffer missing");
		if (j->buf_bytes && (j->G == 0 || j->G > APO_GROUPS_MAX)) return bad(j, "G must be 1..64");
		break;
	case APO_JOB_CANDIDATE_REFS_UPLOAD:               /* buf_bytes = 4 C; C == 0 releases them */
		if (j->buf_bytes && !j->buf) return bad(j, "refs buffer missing");
		if (j->buf_bytes != 4ull * j->C) return bad(j, "refs byte length is not 4 x C");
		break;
	case APO_JOB_TEST_HOOK:
		break;
	default:
		return bad(j, "unknown job kind");
	}
	if (j->kind == APO_JOB_SCORE_HOST || j->kind == APO_JOB_SCORE_HOST_RECORDS || j->kind == APO_JOB_SCORE_HOST_TUPLES) {
		if (j->K > j->C) return bad(j, "K exceeds the number of candidates");
		if (j->corpus_bytes % sizeof(apo_record)) return bad(j, "corpus byte length is not a multiple of 32");
		if (j->corpus_bytes && !j->corpus) return bad(j, "corpus buffer missing");
	}
	if (j->K > 16384) return bad(j, "K exceeds the supported beam width 16384");
	if (j->flags & APO_SCORE_CANDIDATES) {
		if (j->kind != APO_JOB_SCORE_RESIDENT && j->kind != APO_JOB_SCORE_HOST && j->kind != APO_JOB_SCORE_HOST_RECORDS &&
		    j->kind != APO_JOB_SCORE_HOST_TUPLES)
			return bad(j, "the per-candidate breakdown belongs to a scoring call");
		if (j->C == 0) return bad(j, "C must be > 0 for the per-candidate breakdown");
		if (!fits(j->C, sizeof(apo_candidate_report), 1, APO_JOB_CANDIDATES_MAX_BYTES))
			return bad(j, "the per-candidate breakdown of C candidates exceeds 4 GiB");
	}
	if (j->flags & APO_SCORE_CANDIDATE_CORPUS) {
		if (!((j->kind == APO_JOB_SCORE_RESIDENT && j->source == APO_SRC_ROLLOUTS) || j->kind == APO_JOB_SCORE_HOST_RECORDS))
			return bad(j, "the per-candidate corpus reports belong to a scoring call over rollout records");
		if (j->C == 0) return bad(j, "C must be > 0 for the per-candidate corpus reports");
		if (!fits(j->C, sizeof(apo_corpus_report), 1, APO_JOB_CANDIDATE_CORPUS_MAX_BYTES))
			return bad(j, "the per-candidate corpus reports of C candidates exceed 4 GiB");
	}
	if (j->flags & APO_SCORE_CANDIDATE_EXTREMES) {
		if (j->kind != APO_JOB_SCORE_RESIDENT && j->kind != APO_JOB_SCORE_HOST && j->kind != APO_JOB_SCORE_HOST_RECORDS &&
		    j->kind != APO_JOB_SCORE_HOST_TUPLES)
			return bad(j, "the per-candidate extremes belong to a scoring call");
		if (j->C == 0) return bad(j, "C must be > 0 for the per-candidate extremes");
		if (!fits(j->C, sizeof(struct apo_candidate_extremes), 1, APO_JOB_CANDIDATE_EXTREMES_MAX_BYTES))
			return bad(j, "the per-candidate extremes of C candidates exceed 4 GiB");
	}
	if (j->flags & APO_SCORE_CANDIDATE_GROUPS) {
		if (j->kind != APO_JOB_SCORE_RESIDENT && j->kind != APO_JOB_SCORE_HOST && j->kind != APO_JOB_SCORE_HOST_RECORDS &&
		    j->kind != APO_JOB_SCORE_HOST_TUPLES)
			return bad(j, "the per-candidate group scores belong to a scoring call");
		if (j->C == 0) return bad(j, "C must be > 0 for the per-candidate group scores");
		if (j->G == 0 || j->G > APO_GROUPS_MAX) return bad(j, "G must be 1..64 for the per-candidate group scores");
		if (!fits(j->C, j->G, sizeof(apo_group_score), APO_JOB_CANDIDATE_GROUPS_MAX_BYTES))
			return bad(j, "the per-candidate group scores of C candidates and G groups exceed 4 GiB");
	}
	if (j->flags & APO_SCORE_CANDIDATE_SPREAD) {
		if (j->kind != APO_JOB_SCORE_RESIDENT && j->kind != APO_JOB_SCORE_HOST && j->kind != APO_JOB_SCORE_HOST_RECORDS &&
		    j->kind != APO_JOB_SCORE_HOST_TUPLES)
			return bad(j, "the per-candidate reward spreads belong to a scoring call");
		if (j->C == 0) return bad(j, "C must be > 0 for the per-candidate reward spreads");
		if (!fits(j->C, sizeof(struct apo_candidate_spread), 1, APO_JOB_CANDIDATE_SPREAD_MAX_BYTES))
			return bad(j, "the per-candidate reward spreads of C candidates exceed 4 GiB");
	}
	if (j->flags & APO_SCORE_CANDIDATE_PAIRS) {
		if (j->kind != APO_JOB_SCORE_RESIDENT && j->kind != APO_JOB_SCORE_HOST && j->kind != APO_JOB_SCORE_HOST_RECORDS &&
		    j->kind != APO_JOB_SCORE_HOST_TUPLES)
			return bad(j, "the paired comparisons belong to a scoring call");
		if (j->C == 0) return bad(j, "C must be > 0 for the paired comparisons");
		if (!fits(j->C, sizeof(struct apo_candidate_pair), 1, APO_JOB_CANDIDATE_PAIRS_MAX_BYTES))
			return bad(j, "the paired comparisons of C candidates exceed 4 GiB");
	}
	if (j->flags & APO_SCORE_CANDIDATE_GROUP_PAIRS) {
		if (j->kind != APO_JOB_SCORE_RESIDENT && j->kind != APO_JOB_SCORE_HOST && j->kind != APO_JOB_SCORE_HOST_RECORDS &&
		    j->kind != APO_JOB_SCORE_HOST_TUPLES)
			return bad(j, "the paired comparisons per record group belong to a scoring call");
		if (j->C == 0) return bad(j, "C must be > 0 for the paired comparisons per record group");
		if (j->G == 0 || j->G > APO_GROUPS_MAX) return bad(j, "G must be 1..64 for the paired comparisons per record group");
		if (!fits(j->C, j->G, sizeof(struct apo_candidate_pair), APO_JOB_CANDIDATE_GROUP_PAIRS_MAX_BYTES))
			return bad(j, "the paired comparisons per record group of C candidates and G groups exceed 4 GiB");
	}
	return APO_OK;
}

int apo_job_prepare(apo_job *j)
{
	if (j->kind == APO_JOB_SCORE_HOST || j->kind == APO_JOB_SCORE_HOST_RECORDS || j->kind == APO_JOB_SCORE_HOST_TUPLES || j->kind == APO_JOB_SCORE_RESIDENT) {
		/* resident calls learn C from the handle: size for the largest C the handle may hold is unknown here, so the
		 * caller passes C (the count it uploaded); the ABI re-checks K <= C against the loaded shape */
		const uint32_t C = j->C ? j->C : 1, K = j->K ? j->K : 1;
		j->scores = (double *)malloc(8u * (size_t)C); j->counts = (uint64_t *)malloc(8u * (size_t)C); j->topk = (int32_t *)malloc(4u * (size_t)K);
		if (j->flags & APO_SCORE_CANDIDATES) j->candidates = (apo_candidate_report *)malloc(sizeof(apo_candidate_report) * (size_t)C);
		if (j->flags & APO_SCORE_CANDIDATE_CORPUS) j->candidate_corpus = (apo_corpus_report *)malloc(sizeof(apo_corpus_report) * (size_t)C);
		if (j->flags & APO_SCORE_CANDIDATE_EXTREMES)
			j->candidate_extremes = (struct apo_candidate_extremes *)malloc(sizeof(struct apo_candidate_extremes) * (size_t)C);
		if (j->flags & APO_SCORE_CANDIDATE_GROUPS) j->candidate_groups = (apo_group_score *)malloc(sizeof(apo_group_score) * (size_t)C * j->G);
		if (j->flags & APO_SCORE_CANDIDATE_SPREAD)
			j->candidate_spread = (struct apo_candidate_spread *)malloc(sizeof(struct apo_candidate_spread) * (size_t)C);
		if (j->flags & APO_SCORE_CANDIDATE_PAIRS)
			j->candidate_pairs = (struct apo_candidate_pair *)malloc(sizeof(struct apo_candidate_pair) * (size_t)C);
		if (j->flags & APO_SCORE_CANDIDATE_GROUP_PAIRS)
			j->candidate_group_pairs = (struct apo_candidate_pair *)malloc(sizeof(struct apo_candidate_pair) * (size_t)C * j->G);
		if (!j->scores || !j->counts || !j->topk || ((j->flags & APO_SCORE_CANDIDATES) && !j->candidates) ||
		    ((j->flags & APO_SCORE_CANDIDATE_CORPUS) && !j->candidate_corpus) ||
		    ((j->flags & APO_SCORE_CANDIDATE_EXTREMES) && !j->candidate_extremes) ||
		    ((j->flags & APO_SCORE_CANDIDATE_GROUPS) && !j->candidate_groups) ||
		    ((j->flags & APO_SCORE_CANDIDATE_SPREAD) && !j->candidate_spread) ||
		    ((j->flags & APO_SCORE_CANDIDATE_PAIRS) && !j->candidate_pairs) ||
		    ((j->flags & APO_SCORE_CANDIDATE_GROUP_PAIRS) && !j->candidate_group_pairs)) {
			apo_job_release(j); j->rc = APO_E_NOMEM; snprintf(j->err, sizeof j->err, "out of host memory"); return APO_E_NOMEM;
		}
	} else if (j->kind == APO_JOB_REWARD_BATCH) {
		const uint64_t n = j->buf_bytes / sizeof(apo_record);
		j->n_out = n;
		j->dims_out = (double *)malloc(8u * APO_NDIM * (size_t)(n ? n : 1)); j->masks_out = (uint32_t *)malloc(4u * (size_t)(n ? n : 1));
		j->finals_out = (double *)malloc(8u * (size_t)(n ? n : 1));
		if (!j->dims_out || !j->masks_out || !j->finals_out) { apo_job_release(j); j->rc = APO_E_NOMEM; snprintf(j->err, sizeof j->err, "out of host memory"); return APO_E_NOMEM; }
	}
	return APO_OK;
}

void apo_job_release(apo_job *j)
{
	free(j->scores); free(j->counts); free(j->topk); free(j->dims_out); free(j->masks_out); free(j->finals_out); free(j->candidates);
	free(j->candidate_corpus); free(j->candidate_extremes); free(j->candidate_groups); free(j->candidate_spread);
	free(j->candidate_pairs); free(j->candidate_group_pairs);
	j->scores = NULL; j->counts = NULL; j->topk = NULL; j->dims_out = NULL; j->masks_out = NULL; j->finals_out = NULL; j->candidates = NULL;
	j->candidate_corpus = NULL; j->candidate_extremes = NULL; j->candidate_groups = NULL; j->candidate_spread = NULL;
	j->candidate_pairs = NULL; j->candidate_group_pairs = NULL;
}

static void execute(apo_serial *s, apo_job *j)
{
	apo_engine *e = s->e;
	apo_score_opts o; memset(&o, 0, sizeof o);
	o.K = j->K; o.source = j->source; o.flags = j->flags; o.first = j->first; o.count = j->count;
	if (j->kind == APO_JOB_TEST_HOOK) { if (j->hook) j->hook(j->hook_arg); j->rc = APO_OK; return; }
	if (!e) { j->rc = APO_E_STATE; snprintf(j->err, sizeof j->err, "no engine behind this handle"); return; }
	switch (j->kind) {
	case APO_JOB_DIMS_UPLOAD:
		j->rc = j->compact ? apo_dims_upload_compact(e, (const float *)j->buf, j->C, j->T) : apo_dims_upload(e, (const float *)j->buf, j->C, j->T);
		break;
	case APO_JOB_ROLLOUTS_UPLOAD:
		j->rc = j->row_bytes == 16 ? apo_rollouts16_upload(e, (const apo_record16 *)j->buf, j->C, j->T) : apo_rollouts_upload(e, (const apo_record *)j->buf, j->C, j->T);
		break;
	case APO_JOB_CORPUS_UPLOAD:
		j->rc = apo_corpus_upload(e, (const apo_record *)j->buf, j->buf_bytes / sizeof(apo_record), j->idx_base);
		break;
	case APO_JOB_CORPUS_UPLOAD_JSON: {
		uint64_t n = 0;
		j->rc = apo_corpus_upload_json(e, (const char *)j->buf, j->buf_bytes, j->idx_base, &n);
		j->n_out = n;
		break;
	}
	case APO_JOB_SCORE_RESIDENT:
		j->rc = apo_score(e, &o, j->scores, j->counts, j->topk, &j->report);
		break;
	case APO_JOB_SCORE_HOST:
	case APO_JOB_SCORE_HOST_RECORDS:
		o.source = j->kind == APO_JOB_SCORE_HOST ? APO_SRC_DIMS : APO_SRC_ROLLOUTS;
		o.first = 0; o.count = 0;
		j->rc = APO_OK;
		if (j->corpus_bytes) { j->rc = apo_corpus_upload(e, (const apo_record *)j->corpus, j->corpus_bytes / sizeof(apo_record), j->idx_base); o.flags |= APO_SCORE_CORPUS; }
		if (j->rc == APO_OK)
			j->rc = j->kind == APO_JOB_SCORE_HOST
			            ? apo_score_host(e, &o, (const float *)j->buf, j->C, j->T, j->scores, j->counts, j->topk, &j->report)
			            : apo_score_host_records(e, &o, j->buf, j->row_bytes, j->C, j->T, j->scores, j->counts, j->topk, &j->report);
		break;
	case APO_JOB_SCORE_HOST_TUPLES:
		o.source = APO_SRC_DIMS; o.first = 0; o.count = 0;
		j->rc = APO_OK;
		if (j->corpus_bytes) { j->rc = apo_corpus_upload(e, (const apo_record *)j->corpus, j->corpus_bytes / sizeof(apo_record), j->idx_base); o.flags |= APO_SCORE_CORPUS; }
		if (j->rc == APO_OK)
			j->rc = apo_score_host_tuples(e, &o, (const uint16_t *)j->buf, (const uint8_t *)j->aux[0], (const uint32_t *)j->aux[1], (const uint16_t *)j->aux[2],
			                              j->n_tuples, (const uint32_t *)j->aux[3], (const uint32_t *)j->aux[4], j->C, j->T, j->scores, j->counts, j->topk, &j->report);
		break;
	case APO_JOB_REWARD_BATCH:
		j->rc = apo_reward_batch(e, (const apo_record *)j->buf, j->n_out, j->dims_out, j->masks_out, j->finals_out);
		break;
	case APO_JOB_COMM_INIT:
		j->rc = apo_comm_init(e, j->nranks, j->rank, j->comm_id);
		break;
	case APO_JOB_DIMS_TUPLES: {
		uint32_t n = 0;
		j->rc = apo_dims_tuples(e, j->cap, &n);
		j->n_out = n;
		break;
	}
	case APO_JOB_RECORD_GROUPS_UPLOAD:
		j->rc = apo_record_groups_upload(e, (const uint8_t *)j->buf, j->buf_bytes, j->G);
		break;
	case APO_JOB_CANDIDATE_REFS_UPLOAD:
		j->rc = apo_candidate_refs_upload(e, (const uint32_t *)j->buf, j->C);
		break;
	default:
		j->rc = APO_E_ARG;
	}
	if (j->rc == APO_OK && j->candidates) j->rc = apo_candidate_reports(e, 0, j->C, j->candidates);
	if (j->rc == APO_OK && j->candidate_corpus) j->rc = apo_candidate_corpus_reports(e, 0, j->C, j->candidate_corpus);
	if (j->rc == APO_OK && j->candidate_extremes) j->rc = apo_candidate_extremes(e, 0, j->C, j->candidate_extremes);
	if (j->rc == APO_OK && j->candidate_groups) j->rc = apo_candidate_groups(e, 0, j->C, j->G, j->candidate_groups);
	if (j->rc == APO_OK && j->candidate_spread) j->rc = apo_candidate_spread(e, 0, j->C, j->candidate_spread);
	if (j->rc == APO_OK && j->candidate_pairs) j->rc = apo_candidate_pairs(e, 0, j->C, j->candidate_pairs);
	if (j->rc == APO_OK && j->candidate_group_pairs) j->rc = apo_candidate_group_pairs(e, 0, j->C, j->G, j->candidate_group_pairs);
	if (j->rc != APO_OK) snprintf(j->err, sizeof j->err, "%s", apo_last_error(e));
}

void apo_job_run(apo_serial *s, apo_job *j)
{
	pthread_mutex_lock(&s->mu);
	while (s->serving != j->ticket) pthread_cond_wait(&s->cv, &s->mu);
	pthread_mutex_unlock(&s->mu);
	if (j->rc == APO_OK) execute(s, j);              /* a job that failed validation still takes (and releases) its turn */
	pthread_mutex_lock(&s->mu);
	s->serving = j->ticket + 1;
	pthread_cond_broadcast(&s->cv);
	pthread_mutex_unlock(&s->mu);
}
