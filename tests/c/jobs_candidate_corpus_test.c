/* The per-candidate corpus reports in the addon's job core (napi/apo_jobs.c): validation accepts them only on record jobs
 * (scoreResident with source APO_SRC_ROLLOUTS, scoreHostRecords), refuses them without C or when C x sizeof(apo_corpus_report)
 * would exceed APO_JOB_CANDIDATE_CORPUS_MAX_BYTES (no overflow); apo_job_prepare allocates the `candidate_corpus` output
 * only when the flag is set, apo_job_release frees it.  Host-only: no engine is created.
 * Built and run by tests/test_candidate_corpus_cpu.py. */
#include <stdio.h>
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

int main(void)
{
	const uint32_t F = APO_SCORE_CANDIDATE_CORPUS;
	CHECK(sizeof(apo_corpus_report) == 784, "sizeof(apo_corpus_report) = %zu", sizeof(apo_corpus_report));
	CHECK(F == 0x10u && (F & APO_SCORE_CANDIDATES) == 0, "flag value");
	/* accepted on record jobs, and the output exists only with the flag */
	apo_job a = scoring(APO_JOB_SCORE_RESIDENT, APO_SRC_ROLLOUTS, 1000, F);
	CHECK(apo_job_validate(&a) == APO_OK, "resident rollouts job with the flag refused: %s", a.err);
	CHECK(apo_job_prepare(&a) == APO_OK && a.candidate_corpus != NULL && a.candidates == NULL, "candidate_corpus output not allocated alone");
	apo_job_release(&a);
	CHECK(a.candidate_corpus == NULL, "candidate_corpus output not released");
	apo_job b = scoring(APO_JOB_SCORE_RESIDENT, APO_SRC_ROLLOUTS, 1000, APO_SCORE_CANDIDATES);
	CHECK(apo_job_validate(&b) == APO_OK && apo_job_prepare(&b) == APO_OK && b.candidate_corpus == NULL && b.candidates != NULL,
	      "breakdown only: candidate_corpus output allocated");
	apo_job_release(&b);
	apo_job both = scoring(APO_JOB_SCORE_RESIDENT, APO_SRC_ROLLOUTS, 16, F | APO_SCORE_CANDIDATES);
	CHECK(apo_job_validate(&both) == APO_OK && apo_job_prepare(&both) == APO_OK && both.candidate_corpus && both.candidates, "both flags");
	apo_job_release(&both);
	apo_job hr = scoring(APO_JOB_SCORE_HOST_RECORDS, APO_SRC_DIMS, 8, F);
	hr.buf_bytes = 8 * 32;
	CHECK(apo_job_validate(&hr) == APO_OK && apo_job_prepare(&hr) == APO_OK && hr.candidate_corpus, "host records job with the flag: %s", hr.err);
	apo_job_release(&hr);
	/* refused on every job that does not read trace records */
	apo_job d = scoring(APO_JOB_SCORE_RESIDENT, APO_SRC_DIMS, 8, F);
	CHECK(apo_job_validate(&d) == APO_E_ARG && d.err[0], "resident Form D / Q job accepted");
	apo_job t = scoring(APO_JOB_SCORE_RESIDENT, APO_SRC_TUPLES, 8, F);
	CHECK(apo_job_validate(&t) == APO_E_ARG, "resident Form T job accepted");
	apo_job h = scoring(APO_JOB_SCORE_HOST, APO_SRC_DIMS, 8, F);
	CHECK(apo_job_validate(&h) == APO_E_ARG, "host Form D job accepted");
	apo_job ht = scoring(APO_JOB_SCORE_HOST_TUPLES, APO_SRC_DIMS, 8, F);
	CHECK(apo_job_validate(&ht) == APO_E_ARG, "host Form T job accepted");
	apo_job g = scoring(APO_JOB_REWARD_BATCH, APO_SRC_DIMS, 4, F);
	g.buf_bytes = 0; g.buf = NULL;
	CHECK(apo_job_validate(&g) == APO_E_ARG, "reports on a non-scoring job accepted");
	/* the largest C that fits, one more, and a C whose byte count overflows 32 bits */
	const uint32_t cmax = (uint32_t)(APO_JOB_CANDIDATE_CORPUS_MAX_BYTES / sizeof(apo_corpus_report));
	apo_job c = scoring(APO_JOB_SCORE_RESIDENT, APO_SRC_ROLLOUTS, cmax, F);
	CHECK(apo_job_validate(&c) == APO_OK, "C = %u refused", cmax);
	apo_job c1 = scoring(APO_JOB_SCORE_RESIDENT, APO_SRC_ROLLOUTS, cmax + 1, F);
	CHECK(apo_job_validate(&c1) == APO_E_ARG && c1.err[0], "C = %u accepted", cmax + 1);
	apo_job e = scoring(APO_JOB_SCORE_RESIDENT, APO_SRC_ROLLOUTS, 0xFFFFFFFFu, F);
	CHECK(apo_job_validate(&e) == APO_E_ARG, "C = 2^32-1 accepted (C x 784 overflows 32 bits)");
	apo_job z = scoring(APO_JOB_SCORE_RESIDENT, APO_SRC_ROLLOUTS, 0, F);
	CHECK(apo_job_validate(&z) == APO_E_ARG, "C = 0 with the flag accepted");
	if (fails) { printf("%d failure(s)\n", fails); return 1; }
	printf("OK\n");
	return 0;
}
