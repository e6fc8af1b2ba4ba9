/* The paired comparisons in the addon's job core (napi/apo_jobs.c): validation accepts them on every scoring job, refuses them
 * on other jobs, without C, or when C x sizeof(struct apo_candidate_pair) would exceed APO_JOB_CANDIDATE_PAIRS_MAX_BYTES (no
 * overflow); apo_job_prepare allocates the `candidate_pairs` output only when the flag is set, apo_job_release frees it.  The
 * refs upload job refuses a byte length that is not 4 C.  The struct's layout is the one the header states.
 * With the argument "gpu": the same jobs through a real engine — a refs upload job, then resident and host-streaming scoring
 * jobs with the flag return the bytes apo_candidate_pairs gives for the same call.
 * Built and run by tests/test_napi_candidate_pairs.py. */
#include <math.h>
#include <stddef.h>
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
	j.kind = kind; j.source = APO_SRC_DIMS; j.C = C; j.K = 1; j.T = 1; j.flags = flags; j.row_bytes = 32;
	j.buf = dummy; j.buf_bytes = (uint64_t)C * 36;
	return j;
}

static void cpu_checks(void)
{
	const uint32_t F = APO_SCORE_CANDIDATE_PAIRS;
	CHECK(sizeof(struct apo_candidate_pair) == 128, "sizeof(struct apo_candidate_pair) = %zu", sizeof(struct apo_candidate_pair));
	CHECK(offsetof(struct apo_candidate_pair, n) == 8 && offsetof(struct apo_candidate_pair, wins) == 16 &&
	      offsetof(struct apo_candidate_pair, losses) == 24 && offsetof(struct apo_candidate_pair, ties) == 32 &&
	      offsetof(struct apo_candidate_pair, candOnly) == 40 && offsetof(struct apo_candidate_pair, refOnly) == 48 &&
	      offsetof(struct apo_candidate_pair, sumLo) == 56 && offsetof(struct apo_candidate_pair, sumHi) == 64 &&
	      offsetof(struct apo_candidate_pair, sumSq) == 72 && offsetof(struct apo_candidate_pair, meanDiff) == 96 &&
	      offsetof(struct apo_candidate_pair, variance) == 104 && offsetof(struct apo_candidate_pair, stdDev) == 112 &&
	      offsetof(struct apo_candidate_pair, stdErr) == 120, "field offsets");
	CHECK(F == 0x100u && (F & (APO_SCORE_CANDIDATES | APO_SCORE_CANDIDATE_CORPUS | APO_SCORE_CANDIDATE_EXTREMES | APO_SCORE_CANDIDATE_GROUPS |
	                           APO_SCORE_CANDIDATE_SPREAD)) == 0, "flag value");
	CHECK(APO_JOB_CANDIDATE_REFS_UPLOAD == APO_JOB_RECORD_GROUPS_UPLOAD + 1, "refs upload job appended to the enum");
	const apo_job_kind kinds[4] = {APO_JOB_SCORE_RESIDENT, APO_JOB_SCORE_HOST, APO_JOB_SCORE_HOST_RECORDS, APO_JOB_SCORE_HOST_TUPLES};
	for (int k = 0; k < 4; k++) {
		apo_job a = scoring(kinds[k], 100, F);
		if (kinds[k] == APO_JOB_SCORE_HOST_RECORDS) a.buf_bytes = 100 * 32;
		if (kinds[k] == APO_JOB_SCORE_HOST_TUPLES) {
			static uint32_t book[8 * 256], d2book[4096], pc[1];
			static uint16_t pd[1];
			static uint8_t th[100];
			a.buf_bytes = 100 * 2; a.aux[0] = th; a.aux_bytes[0] = 100; a.n_tuples = 1;
			a.aux[1] = pc; a.aux_bytes[1] = 4; a.aux[2] = pd; a.aux_bytes[2] = 2;
			a.aux[3] = book; a.aux_bytes[3] = sizeof book; a.aux[4] = d2book; a.aux_bytes[4] = sizeof d2book;
		}
		CHECK(apo_job_validate(&a) == APO_OK, "scoring job %d with the flag refused: %s", k, a.err);
		CHECK(apo_job_prepare(&a) == APO_OK && a.candidate_pairs != NULL && a.candidates == NULL && a.candidate_spread == NULL &&
		      a.candidate_groups == NULL, "candidate_pairs output not allocated alone (job %d)", k);
		apo_job_release(&a);
		CHECK(a.candidate_pairs == NULL, "candidate_pairs output not released");
	}
	apo_job b = scoring(APO_JOB_SCORE_RESIDENT, 100, APO_SCORE_CANDIDATE_SPREAD);
	CHECK(apo_job_validate(&b) == APO_OK && apo_job_prepare(&b) == APO_OK && b.candidate_pairs == NULL, "spread only: pairs allocated");
	apo_job_release(&b);
	apo_job g = scoring(APO_JOB_REWARD_BATCH, 4, F);
	g.buf_bytes = 0; g.buf = NULL;
	CHECK(apo_job_validate(&g) == APO_E_ARG && g.err[0], "pairs on a non-scoring job accepted");
	/* the largest C that fits, one more, and a C whose byte count passes 32 bits */
	const uint32_t cmax = (uint32_t)(APO_JOB_CANDIDATE_PAIRS_MAX_BYTES / sizeof(struct apo_candidate_pair));
	apo_job c = scoring(APO_JOB_SCORE_RESIDENT, cmax, F);
	CHECK(apo_job_validate(&c) == APO_OK, "C = %u refused", cmax);
	apo_job c1 = scoring(APO_JOB_SCORE_RESIDENT, cmax + 1, F);
	CHECK(apo_job_validate(&c1) == APO_E_ARG && c1.err[0], "C = %u accepted", cmax + 1);
	apo_job e = scoring(APO_JOB_SCORE_RESIDENT, 0xFFFFFFFFu, F);
	CHECK(apo_job_validate(&e) == APO_E_ARG, "C = 2^32-1 accepted");
	apo_job z = scoring(APO_JOB_SCORE_RESIDENT, 0, F);
	CHECK(apo_job_validate(&z) == APO_E_ARG, "C = 0 with the flag accepted");
	/* the refs upload job: 4 C bytes, a buffer when C > 0, C == 0 releases */
	static uint32_t refs[3] = {1, 0, APO_PAIR_NONE};
	apo_job u; memset(&u, 0, sizeof u);
	u.kind = APO_JOB_CANDIDATE_REFS_UPLOAD; u.buf = refs; u.buf_bytes = sizeof refs; u.C = 3;
	CHECK(apo_job_validate(&u) == APO_OK, "refs upload refused: %s", u.err);
	u.rc = APO_OK; u.buf_bytes = 10;
	CHECK(apo_job_validate(&u) == APO_E_ARG, "refs of 10 bytes for C = 3 accepted");
	u.rc = APO_OK; u.buf = NULL; u.buf_bytes = 12;
	CHECK(apo_job_validate(&u) == APO_E_ARG, "refs upload without a buffer accepted");
	u.rc = APO_OK; u.buf_bytes = 0; u.C = 0;
	CHECK(apo_job_validate(&u) == APO_OK, "refs release refused: %s", u.err);
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
	unsigned x = 993u;
	for (size_t i = 0; i < (size_t)C * T * 9; i++) {
		x = x * 1103515245u + 12345u;
		const unsigned r = (x >> 8) % 10u;
		dims[i] = r == 0 ? NAN : (r < 4 ? -1.0f : (r < 7 ? 1.0f : 0.5f));
	}
	apo_job up; memset(&up, 0, sizeof up);
	up.kind = APO_JOB_DIMS_UPLOAD; up.buf = dims; up.buf_bytes = sizeof(float) * C * T * 9; up.C = C; up.T = T;
	CHECK(run(s, &up) == APO_OK, "dimsUpload: %s", up.err);
	apo_job_release(&up);

	uint32_t refs[C] = {APO_PAIR_NONE, 0, 0, 4, 5, 5};
	apo_job u; memset(&u, 0, sizeof u);
	u.kind = APO_JOB_CANDIDATE_REFS_UPLOAD; u.buf = refs; u.buf_bytes = sizeof refs; u.C = C;
	CHECK(run(s, &u) == APO_OK, "candidateRefsUpload: %s", u.err);
	static struct apo_candidate_pair direct[C];
	apo_job r = scoring(APO_JOB_SCORE_RESIDENT, C, APO_SCORE_CANDIDATE_PAIRS);
	r.buf = NULL; r.buf_bytes = 0; r.K = 2;
	CHECK(run(s, &r) == APO_OK && r.candidate_pairs, "scoreResident with candidatePairs: %s", r.err);
	CHECK(apo_candidate_pairs(s->e, 0, C, direct) == APO_OK, "apo_candidate_pairs after the job");
	CHECK(r.candidate_pairs && memcmp(direct, r.candidate_pairs, sizeof direct) == 0, "job pairs != apo_candidate_pairs");
	for (int c = 0; r.candidate_pairs && c < C; c++) {
		CHECK(direct[c].ref == refs[c], "ref of candidate %d", c);
		if (refs[c] == APO_PAIR_NONE) { CHECK(direct[c].n == 0 && isnan(direct[c].meanDiff), "candidate %d without a reference", c); continue; }
		CHECK(direct[c].n + direct[c].candOnly == r.counts[c] && direct[c].n + direct[c].refOnly == r.counts[refs[c]], "counts of %d", c);
		CHECK(direct[c].wins + direct[c].losses + direct[c].ties == direct[c].n, "tallies of %d", c);
	}
	CHECK(direct[5].ties == direct[5].n && direct[5].sumLo == 0 && direct[5].sumHi == 0, "self-pair");
	apo_job h = scoring(APO_JOB_SCORE_HOST, C, APO_SCORE_CANDIDATE_PAIRS | APO_SCORE_CANDIDATE_SPREAD);
	h.buf = dims; h.buf_bytes = sizeof(float) * C * T * 9; h.T = T; h.K = 2;
	CHECK(run(s, &h) == APO_OK && h.candidate_pairs && h.candidate_spread, "score (host) with candidatePairs: %s", h.err);
	CHECK(h.candidate_pairs && memcmp(h.candidate_pairs, direct, sizeof direct) == 0, "host-streamed pairs != resident");
	apo_job n = scoring(APO_JOB_SCORE_RESIDENT, C, 0);
	n.buf = NULL; n.buf_bytes = 0; n.K = 2;
	CHECK(run(s, &n) == APO_OK && n.candidate_pairs == NULL, "flag clear: %s", n.err);
	CHECK(apo_candidate_pairs(s->e, 0, C, direct) == APO_E_STATE, "pairs readable after a flag-clear call");
	apo_job rel; memset(&rel, 0, sizeof rel);
	rel.kind = APO_JOB_CANDIDATE_REFS_UPLOAD; rel.C = 0;
	CHECK(run(s, &rel) == APO_OK, "refs release: %s", rel.err);
	apo_job q = scoring(APO_JOB_SCORE_RESIDENT, C, APO_SCORE_CANDIDATE_PAIRS);
	q.buf = NULL; q.buf_bytes = 0; q.K = 2;
	CHECK(run(s, &q) == APO_E_STATE, "pairs without refs accepted");
	apo_job_release(&u); apo_job_release(&r); apo_job_release(&h); apo_job_release(&n); apo_job_release(&rel); apo_job_release(&q);
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
