/*
 * cand_oracle.c — CPU oracle of the per-candidate breakdown (apo_candidate_report, APO_SCORE_CANDIDATES).
 *
 * TEST INFRASTRUCTURE ONLY (as apo_oracle.h).  Per candidate c, over the evaluations [0, T) of its row:
 *   - feedback tally (APO:509-516): Form D from d0 (TCS:677-679: 1 good, -1 bad, else none, absent included);
 *     Form R from the feedback field (1 good, 2 bad, else none, VALID or not);
 *   - over evaluations with a non-null finalReward (TCS:784 / APO:550): the exact integer sum of rint(fr * 2^52) and, per
 *     present dimension, of rint(v * 2^52) with v the fp32 value widened (Form D) or the binary64 TCS:668-763 value
 *     (Form R), as __int128, and the counts;
 *   - the first three record positions (idx_base + t, ascending) whose tally is 'bad';
 *   - refused = 1 when such an evaluation has a present dimension with |v| >= 2048 (+-inf included): rint(v * 2^52) does not fit in
 *     int64 there (llrint's result is unspecified), so the term is left out and the engine fails the call with APO_E_ARG.
 * Rounding to binary64 and the report rules are applied by oracle/candidates.py.
 */
#include <math.h>
#include <pthread.h>
#include <stdlib.h>
#include <string.h>
#include "apo_oracle.h"
#include "cand_oracle.h"

static const double kFx = 4503599627370496.0;   /* 2^52 */
static const double kFxBound = 2048.0;           /* |v| < 2^11 <=> |rint(v * 2^52)| < 2^63 */

typedef struct {
	uint64_t total, good, bad, withReward;
	__int128 rew, dim[ORC_NDIM];
	uint64_t dimCount[ORC_NDIM];
	int64_t ex[3]; int nex;
	int refused;
} acc_t;

static void acc_zero(acc_t *a) { memset(a, 0, sizeof *a); for (int k = 0; k < 3; k++) a->ex[k] = -1; }

/* one evaluation: dims (NaN = absent), non-null finalReward or not, tally 0 none / 1 good / 2 bad */
static void acc_eval(acc_t *a, const double d[ORC_NDIM], int valid, double fr, int tally, int64_t pos) {
	a->total++;
	if (tally == 1) a->good++;
	if (tally == 2) { a->bad++; if (a->nex < 3) a->ex[a->nex++] = pos; }
	if (!valid) return;
	a->withReward++;
	a->rew += (__int128)llrint(fr * kFx);
	for (int i = 0; i < ORC_NDIM; i++) {
		if (d[i] != d[i]) continue;                                         /* absent */
		if (!(fabs(d[i]) < kFxBound)) { a->refused = 1; continue; }
		a->dim[i] += (__int128)llrint(d[i] * kFx); a->dimCount[i]++;
	}
}

/* b follows a on the record axis */
static void acc_merge(acc_t *a, const acc_t *b) {
	a->total += b->total; a->good += b->good; a->bad += b->bad; a->withReward += b->withReward; a->rew += b->rew;
	for (int i = 0; i < ORC_NDIM; i++) { a->dim[i] += b->dim[i]; a->dimCount[i] += b->dimCount[i]; }
	for (int k = 0; k < b->nex && a->nex < 3; k++) a->ex[a->nex++] = b->ex[k];
	a->refused |= b->refused;
}

static void acc_out(const acc_t *a, orc_cand_fx *o) {
	o->total = a->total; o->good = a->good; o->bad = a->bad; o->none = a->total - a->good - a->bad; o->withReward = a->withReward;
	o->rew_lo = (uint64_t)a->rew; o->rew_hi = (int64_t)(a->rew >> 64);
	for (int i = 0; i < ORC_NDIM; i++) {
		o->dim_lo[i] = (uint64_t)a->dim[i]; o->dim_hi[i] = (int64_t)(a->dim[i] >> 64); o->dim_count[i] = a->dimCount[i];
	}
	for (int k = 0; k < 3; k++) o->badExamples[k] = a->ex[k];
	o->refused = (uint32_t)a->refused; o->pad = 0;
}

static void eval_row(acc_t *a, const float row[ORC_NDIM], const double w[ORC_NDIM], int64_t pos) {
	double d[ORC_NDIM], fr = 0.0;
	for (int i = 0; i < ORC_NDIM; i++) d[i] = (double)row[i];
	const int valid = orc_final_reward_f32(row, w, &fr);
	const int tally = d[0] == 1.0 ? 1 : (d[0] == -1.0 ? 2 : 0);    /* NaN (absent) compares unequal: none */
	acc_eval(a, d, valid, fr, tally, pos);
}

static void eval_record(acc_t *a, const orc_record *r, const double w[ORC_NDIM], int64_t pos) {
	double d[ORC_NDIM], fr = 0.0;
	const uint32_t mask = orc_reward_dims(r, d);
	const int valid = (r->flags & ORC_F_VALID) && orc_final_reward(d, mask, w, &fr);
	const int tally = r->feedback == 1 ? 1 : (r->feedback == 2 ? 2 : 0);   /* VALID or not, as the corpus scan counts */
	acc_eval(a, d, valid, fr, tally, pos);
}

void orc_cand_dims(const float *dims, uint32_t C, uint64_t T, uint64_t pitch_evals, uint64_t idx_base, const double w[ORC_NDIM],
                   orc_cand_fx *out) {
	for (uint32_t c = 0; c < C; c++) {
		acc_t a; acc_zero(&a);
		for (uint64_t t = 0; t < T; t++) eval_row(&a, dims + ((uint64_t)c * pitch_evals + t) * ORC_NDIM, w, (int64_t)(idx_base + t));
		acc_out(&a, out + c);
	}
}

void orc_cand_records(const orc_record *recs, uint32_t C, uint64_t T, uint64_t pitch, uint64_t idx_base, const double w[ORC_NDIM],
                      orc_cand_fx *out) {
	for (uint32_t c = 0; c < C; c++) {
		acc_t a; acc_zero(&a);
		for (uint64_t t = 0; t < T; t++) eval_record(&a, recs + (uint64_t)c * pitch + t, w, (int64_t)(idx_base + t));
		acc_out(&a, out + c);
	}
}

typedef struct {
	uint64_t seed, t0, t1; uint32_t c, agent_permille; int records; const double *w; acc_t acc;
} gen_job;

static void *gen_worker(void *p) {
	gen_job *j = (gen_job *)p;
	acc_zero(&j->acc);
	float row[ORC_NDIM];
	orc_record r;
	for (uint64_t t = j->t0; t < j->t1; t++) {
		if (j->records) {
			orc_gen_record(j->seed, ORC_STREAM_ROLLOUT, j->c, t, j->agent_permille, &r);
			eval_record(&j->acc, &r, j->w, (int64_t)t);
		} else {
			orc_gen_dims_row(j->seed, j->c, t, j->agent_permille, row);
			eval_row(&j->acc, row, j->w, (int64_t)t);
		}
	}
	return NULL;
}

static void cand_generated(int records, uint64_t seed, const uint32_t *cands, uint32_t ncand, uint64_t t0, uint64_t T,
                           uint32_t agent_permille, const double w[ORC_NDIM], orc_cand_fx *out, int nthreads) {
	if (nthreads < 1) nthreads = 1;
	if (nthreads > 256) nthreads = 256;
	gen_job *jobs = (gen_job *)calloc((size_t)nthreads, sizeof(gen_job));
	pthread_t *th = (pthread_t *)calloc((size_t)nthreads, sizeof(pthread_t));
	for (uint32_t k = 0; k < ncand; k++) {
		for (int i = 0; i < nthreads; i++) {
			gen_job *j = &jobs[i];
			j->seed = seed; j->c = cands[k]; j->agent_permille = agent_permille; j->records = records; j->w = w;
			j->t0 = t0 + T * (uint64_t)i / (uint64_t)nthreads;
			j->t1 = t0 + T * (uint64_t)(i + 1) / (uint64_t)nthreads;
			if (i > 0 && pthread_create(&th[i], NULL, gen_worker, j) != 0) { th[i] = 0; gen_worker(j); }
		}
		gen_worker(&jobs[0]);
		for (int i = 1; i < nthreads; i++) if (th[i]) pthread_join(th[i], NULL);
		acc_t a; acc_zero(&a);
		for (int i = 0; i < nthreads; i++) acc_merge(&a, &jobs[i].acc);   /* slice order = record order */
		acc_out(&a, out + k);
	}
	free(jobs); free(th);
}

void orc_cand_generated(uint64_t seed, const uint32_t *cands, uint32_t ncand, uint64_t t0, uint64_t T, uint32_t agent_permille,
                        const double w[ORC_NDIM], orc_cand_fx *out, int nthreads) {
	cand_generated(0, seed, cands, ncand, t0, T, agent_permille, w, out, nthreads);
}

void orc_cand_generated_records(uint64_t seed, const uint32_t *cands, uint32_t ncand, uint64_t t0, uint64_t T, uint32_t agent_permille,
                                const double w[ORC_NDIM], orc_cand_fx *out, int nthreads) {
	cand_generated(1, seed, cands, ncand, t0, T, agent_permille, w, out, nthreads);
}
