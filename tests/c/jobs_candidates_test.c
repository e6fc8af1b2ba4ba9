/* The per-candidate breakdown in the addon's job core (napi/apo_jobs.c): validation refuses a breakdown outside a scoring
 * call, without C, or whose C x sizeof(apo_candidate_report) block would exceed APO_JOB_CANDIDATES_MAX_BYTES (no overflow);
 * apo_job_prepare allocates the `candidates` output only when the flag is set, apo_job_release frees it.
 * With the argument "gpu": the same jobs through a real engine — a resident and a host-streaming scoring job with the flag
 * hand back the breakdown apo_candidate_reports gives for the same call, and the flag-clear job none.
 * Built and run by tests/test_napi_candidates.py. */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "apo_jobs.h"

static int fails;
#define CHECK(cond, ...) do { if (!(cond)) { printf("FAIL: "); printf(__VA_ARGS__); printf("\n"); fails++; } } while (0)

static apo_job scoring(apo_job_kind kind, uint32_t C, uint32_t flags)
{
	static float dummy[36];
	apo_job j; memset(&j, 0, sizeof j);
	j.kind = kind; j.C = C; j.K = 1; j.T = 1; j.flags = flags; j.row_bytes = 32;
	j.buf = dummy; j.buf_bytes = (uint64_t)C * 36;
	return j;
}

static int cpu_checks(void)
{
	CHECK(sizeof(apo_candidate_report) == 376, "sizeof(apo_candidate_report) = %zu", sizeof(apo_candidate_report));
	/* accepted, and the output exists only with the flag */
	apo_job a = scoring(APO_JOB_SCORE_RESIDENT, 1000, APO_SCORE_CANDIDATES);
	CHECK(apo_job_validate(&a) == APO_OK, "resident job with the flag refused: %s", a.err);
	CHECK(apo_job_prepare(&a) == APO_OK && a.candidates != NULL, "no candidates output allocated");
	apo_job_release(&a);
	CHECK(a.candidates == NULL, "candidates output not released");
	apo_job b = scoring(APO_JOB_SCORE_RESIDENT, 1000, APO_SCORE_CORPUS);
	CHECK(apo_job_validate(&b) == APO_OK && apo_job_prepare(&b) == APO_OK && b.candidates == NULL, "flag clear: candidates output allocated");
	apo_job_release(&b);
	/* the largest C that fits, and one more */
	const uint32_t cmax = (uint32_t)(APO_JOB_CANDIDATES_MAX_BYTES / sizeof(apo_candidate_report));
	apo_job c = scoring(APO_JOB_SCORE_RESIDENT, cmax, APO_SCORE_CANDIDATES);
	CHECK(apo_job_validate(&c) == APO_OK, "C = %u refused", cmax);
	apo_job d = scoring(APO_JOB_SCORE_RESIDENT, cmax + 1, APO_SCORE_CANDIDATES);
	CHECK(apo_job_validate(&d) == APO_E_ARG && d.err[0], "C = %u accepted", cmax + 1);
	apo_job e = scoring(APO_JOB_SCORE_RESIDENT, 0xFFFFFFFFu, APO_SCORE_CANDIDATES);
	CHECK(apo_job_validate(&e) == APO_E_ARG, "C = 2^32-1 accepted (C x 376 overflows 32 bits)");
	apo_job f = scoring(APO_JOB_SCORE_RESIDENT, 0, APO_SCORE_CANDIDATES);
	CHECK(apo_job_validate(&f) == APO_E_ARG, "C = 0 with the flag accepted");
	apo_job g = scoring(APO_JOB_REWARD_BATCH, 4, APO_SCORE_CANDIDATES);
	g.buf_bytes = 0; g.buf = NULL;
	CHECK(apo_job_validate(&g) == APO_E_ARG, "breakdown on a non-scoring job accepted");
	/* host-streaming kinds take it too; an oversized one is refused before any allocation */
	apo_job h = scoring(APO_JOB_SCORE_HOST, 8, APO_SCORE_CANDIDATES);
	CHECK(apo_job_validate(&h) == APO_OK && apo_job_prepare(&h) == APO_OK && h.candidates, "host job with the flag");
	apo_job_release(&h);
	apo_job k = scoring(APO_JOB_SCORE_HOST_RECORDS, 8, APO_SCORE_CANDIDATES);
	k.buf_bytes = 8 * 32;
	CHECK(apo_job_validate(&k) == APO_OK, "records job with the flag refused: %s", k.err);
	return fails;
}

static int run(apo_serial *s, apo_job *j)
{
	if (apo_job_validate(j) == APO_OK) apo_job_prepare(j);
	j->ticket = apo_serial_ticket(s);
	apo_job_run(s, j);
	return j->rc;
}

static int gpu_checks(void)
{
	char err[256];
	apo_serial *s = apo_serial_create(0, err, sizeof err);
	if (!s) { printf("FAIL: no engine: %s\n", err); return 1; }
	enum { C = 6, T = 5000 };
	float *dims = (float *)malloc(sizeof(float) * C * T * 9);
	unsigned x = 12345u;
	for (size_t i = 0; i < (size_t)C * T * 9; i++) {
		x = x * 1103515245u + 12345u;
		const unsigned r = (x >> 8) % 10u;
		dims[i] = r == 0 ? NAN : (r < 4 ? -1.0f : (r < 7 ? 1.0f : 0.5f));
	}
	apo_job up; memset(&up, 0, sizeof up);
	up.kind = APO_JOB_DIMS_UPLOAD; up.buf = dims; up.buf_bytes = sizeof(float) * C * T * 9; up.C = C; up.T = T;
	CHECK(run(s, &up) == APO_OK, "dimsUpload: %s", up.err);
	apo_job_release(&up);

	apo_candidate_report direct[C];
	apo_job r = scoring(APO_JOB_SCORE_RESIDENT, C, APO_SCORE_CANDIDATES);
	r.buf = NULL; r.buf_bytes = 0; r.K = 2;
	CHECK(run(s, &r) == APO_OK && r.candidates, "scoreResident with candidates: %s", r.err);
	CHECK(apo_candidate_reports(s->e, 0, C, direct) == APO_OK, "apo_candidate_reports after the job");
	CHECK(r.candidates && memcmp(direct, r.candidates, sizeof direct) == 0, "job breakdown != apo_candidate_reports");
	for (int c = 0; r.candidates && c < C; c++) {
		CHECK(r.candidates[c].withReward == r.counts[c], "withReward != counts[%d]", c);
		CHECK(r.candidates[c].withReward == 0 || memcmp(&r.candidates[c].avgReward, &r.scores[c], 8) == 0, "avgReward != scores[%d]", c);
	}
	apo_job h = scoring(APO_JOB_SCORE_HOST, C, APO_SCORE_CANDIDATES);
	h.buf = dims; h.buf_bytes = sizeof(float) * C * T * 9; h.T = T; h.K = 2;
	CHECK(run(s, &h) == APO_OK && h.candidates, "score (host) with candidates: %s", h.err);
	CHECK(h.candidates && r.candidates && memcmp(h.candidates, r.candidates, sizeof direct) == 0, "host-streamed breakdown != resident");
	apo_job n = scoring(APO_JOB_SCORE_RESIDENT, C, 0);
	n.buf = NULL; n.buf_bytes = 0; n.K = 2;
	CHECK(run(s, &n) == APO_OK && n.candidates == NULL, "flag clear: %s", n.err);
	CHECK(apo_candidate_reports(s->e, 0, C, direct) == APO_E_STATE, "breakdown readable after a flag-clear call");
	apo_job_release(&r); apo_job_release(&h); apo_job_release(&n);
	apo_serial_destroy(s);
	free(dims);
	return fails;
}

int main(int argc, char **argv)
{
	cpu_checks();
	if (argc > 1 && strcmp(argv[1], "gpu") == 0) gpu_checks();
	if (fails) return 1;
	printf("OK\n");
	return 0;
}
