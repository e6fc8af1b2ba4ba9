/* The per-candidate extremes in the addon's job core (napi/apo_jobs.c): validation accepts them on every scoring job,
 * refuses them on other jobs, without C, or when C x sizeof(struct apo_candidate_extremes) would exceed
 * APO_JOB_CANDIDATE_EXTREMES_MAX_BYTES (no overflow); apo_job_prepare allocates the `candidate_extremes` output only when the
 * flag is set, apo_job_release frees it.
 * With the argument "gpu": the same jobs through a real engine — resident and host-streaming scoring jobs with the flag return
 * the bytes apo_candidate_extremes gives for the same call, with and without the other two per-candidate flags.
 * Built and run by tests/test_napi_candidate_extremes.py. */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "apo_jobs.h"

static int fails;
#define CHECK(cond, ...) do { if (!(cond)) { printf("FAIL: "); printf(__VA_ARGS__); printf("\n"); fails++; } } while (0)

static apo_job scoring(apo_job_kind kind, uint32_t source, uint32_t C, uint32_t flags)
{
	static float dummy[36];
	apo_job j; memset(&j, 0, sizeof j);
	j.kind = kind; j.source = source; j.C = C; j.K = 1; j.T = 1; j.flags = flags; j.row_bytes = 32;
	j.buf = dummy; j.buf_bytes = (uint64_t)C * 36;
	return j;
}

static void cpu_checks(void)
{
	const uint32_t F = APO_SCORE_CANDIDATE_EXTREMES;
	CHECK(sizeof(struct apo_candidate_extremes) == 1032, "sizeof(struct apo_candidate_extremes) = %zu", sizeof(struct apo_candidate_extremes));
	CHECK(F == 0x20u && (F & (APO_SCORE_CANDIDATES | APO_SCORE_CANDIDATE_CORPUS)) == 0, "flag value");
	/* accepted on every scoring job, and the output exists only with the flag */
	const apo_job_kind kinds[4] = {APO_JOB_SCORE_RESIDENT, APO_JOB_SCORE_HOST, APO_JOB_SCORE_HOST_RECORDS, APO_JOB_SCORE_HOST_TUPLES};
	for (int k = 0; k < 4; k++) {
		apo_job a = scoring(kinds[k], APO_SRC_DIMS, 100, F);
		if (kinds[k] == APO_JOB_SCORE_HOST_RECORDS) a.buf_bytes = 100 * 32;
		if (kinds[k] == APO_JOB_SCORE_HOST_TUPLES) {                 /* one evaluation per candidate, a one-entry dictionary */
			static uint32_t book[8 * 256], d2book[4096], pc[1];
			static uint16_t pd[1];
			static uint8_t th[100];
			a.buf_bytes = 100 * 2; a.aux[0] = th; a.aux_bytes[0] = 100; a.n_tuples = 1;
			a.aux[1] = pc; a.aux_bytes[1] = 4; a.aux[2] = pd; a.aux_bytes[2] = 2;
			a.aux[3] = book; a.aux_bytes[3] = sizeof book; a.aux[4] = d2book; a.aux_bytes[4] = sizeof d2book;
		}
		CHECK(apo_job_validate(&a) == APO_OK, "scoring job %d with the flag refused: %s", k, a.err);
		CHECK(apo_job_prepare(&a) == APO_OK && a.candidate_extremes != NULL && a.candidates == NULL && a.candidate_corpus == NULL,
		      "candidate_extremes output not allocated alone (job %d)", k);
		apo_job_release(&a);
		CHECK(a.candidate_extremes == NULL, "candidate_extremes output not released");
	}
	apo_job b = scoring(APO_JOB_SCORE_RESIDENT, APO_SRC_DIMS, 100, APO_SCORE_CANDIDATES);
	CHECK(apo_job_validate(&b) == APO_OK && apo_job_prepare(&b) == APO_OK && b.candidate_extremes == NULL, "breakdown only: extremes allocated");
	apo_job_release(&b);
	apo_job all = scoring(APO_JOB_SCORE_RESIDENT, APO_SRC_ROLLOUTS, 16, F | APO_SCORE_CANDIDATES | APO_SCORE_CANDIDATE_CORPUS);
	CHECK(apo_job_validate(&all) == APO_OK && apo_job_prepare(&all) == APO_OK && all.candidate_extremes && all.candidates && all.candidate_corpus,
	      "all three flags");
	apo_job_release(&all);
	apo_job g = scoring(APO_JOB_REWARD_BATCH, APO_SRC_DIMS, 4, F);
	g.buf_bytes = 0; g.buf = NULL;
	CHECK(apo_job_validate(&g) == APO_E_ARG && g.err[0], "extremes on a non-scoring job accepted");
	/* the largest C that fits, one more, and a C whose byte count overflows 32 bits */
	const uint32_t cmax = (uint32_t)(APO_JOB_CANDIDATE_EXTREMES_MAX_BYTES / sizeof(struct apo_candidate_extremes));
	apo_job c = scoring(APO_JOB_SCORE_RESIDENT, APO_SRC_DIMS, cmax, F);
	CHECK(apo_job_validate(&c) == APO_OK, "C = %u refused", cmax);
	apo_job c1 = scoring(APO_JOB_SCORE_RESIDENT, APO_SRC_DIMS, cmax + 1, F);
	CHECK(apo_job_validate(&c1) == APO_E_ARG && c1.err[0], "C = %u accepted", cmax + 1);
	apo_job e = scoring(APO_JOB_SCORE_RESIDENT, APO_SRC_DIMS, 0xFFFFFFFFu, F);
	CHECK(apo_job_validate(&e) == APO_E_ARG, "C = 2^32-1 accepted (C x 1032 overflows 32 bits)");
	apo_job z = scoring(APO_JOB_SCORE_RESIDENT, APO_SRC_DIMS, 0, F);
	CHECK(apo_job_validate(&z) == APO_E_ARG, "C = 0 with the flag accepted");
}

static int run(apo_serial *s, apo_job *j)
{
	if (apo_job_validate(j) == APO_OK) apo_job_prepare(j);
	j->ticket = apo_serial_ticket(s);
	apo_job_run(s, j);
	return j->rc;
}

static void gpu_checks(void)
{
	char err[256];
	apo_serial *s = apo_serial_create(0, err, sizeof err);
	if (!s) { printf("FAIL: no engine: %s\n", err); fails++; return; }
	enum { C = 6, T = 5000 };
	float *dims = (float *)malloc(sizeof(float) * C * T * 9);
	unsigned x = 777u;
	for (size_t i = 0; i < (size_t)C * T * 9; i++) {
		x = x * 1103515245u + 12345u;
		const unsigned r = (x >> 8) % 10u;
		dims[i] = r == 0 ? NAN : (r < 4 ? -1.0f : (r < 7 ? 1.0f : 0.5f));
	}
	apo_job up; memset(&up, 0, sizeof up);
	up.kind = APO_JOB_DIMS_UPLOAD; up.buf = dims; up.buf_bytes = sizeof(float) * C * T * 9; up.C = C; up.T = T;
	CHECK(run(s, &up) == APO_OK, "dimsUpload: %s", up.err);
	apo_job_release(&up);

	static struct apo_candidate_extremes direct[C];
	apo_job r = scoring(APO_JOB_SCORE_RESIDENT, APO_SRC_DIMS, C, APO_SCORE_CANDIDATE_EXTREMES);
	r.buf = NULL; r.buf_bytes = 0; r.K = 2;
	CHECK(run(s, &r) == APO_OK && r.candidate_extremes, "scoreResident with candidateExtremes: %s", r.err);
	CHECK(apo_candidate_extremes(s->e, 0, C, direct) == APO_OK, "apo_candidate_extremes after the job");
	CHECK(r.candidate_extremes && memcmp(direct, r.candidate_extremes, sizeof direct) == 0, "job extremes != apo_candidate_extremes");
	for (int c = 0; r.candidate_extremes && c < C; c++)
		CHECK(r.candidate_extremes[c].n == (r.counts[c] < 32 ? r.counts[c] : 32), "n != min(32, counts[%d])", c);
	apo_job b = scoring(APO_JOB_SCORE_RESIDENT, APO_SRC_DIMS, C, APO_SCORE_CANDIDATE_EXTREMES | APO_SCORE_CANDIDATES);
	b.buf = NULL; b.buf_bytes = 0; b.K = 2;
	CHECK(run(s, &b) == APO_OK && b.candidate_extremes && b.candidates, "scoreResident with both flags: %s", b.err);
	CHECK(b.candidate_extremes && memcmp(direct, b.candidate_extremes, sizeof direct) == 0, "extremes differ beside the breakdown");
	apo_job h = scoring(APO_JOB_SCORE_HOST, APO_SRC_DIMS, C, APO_SCORE_CANDIDATE_EXTREMES);
	h.buf = dims; h.buf_bytes = sizeof(float) * C * T * 9; h.T = T; h.K = 2;
	CHECK(run(s, &h) == APO_OK && h.candidate_extremes, "score (host) with candidateExtremes: %s", h.err);
	CHECK(h.candidate_extremes && memcmp(h.candidate_extremes, direct, sizeof direct) == 0, "host-streamed extremes != resident");
	apo_job n = scoring(APO_JOB_SCORE_RESIDENT, APO_SRC_DIMS, C, 0);
	n.buf = NULL; n.buf_bytes = 0; n.K = 2;
	CHECK(run(s, &n) == APO_OK && n.candidate_extremes == NULL, "flag clear: %s", n.err);
	CHECK(apo_candidate_extremes(s->e, 0, C, direct) == APO_E_STATE, "extremes readable after a flag-clear call");
	apo_job_release(&r); apo_job_release(&b); apo_job_release(&h); apo_job_release(&n);
	apo_serial_destroy(s);
	free(dims);
}

int main(int argc, char **argv)
{
	cpu_checks();
	if (argc > 1 && strcmp(argv[1], "gpu") == 0) gpu_checks();
	if (fails) { printf("%d failure(s)\n", fails); return 1; }
	printf("OK\n");
	return 0;
}
