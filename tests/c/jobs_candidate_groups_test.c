/* The per-candidate group scores in the addon's job core (napi/apo_jobs.c): validation accepts them on every scoring job with
 * 1 <= G <= APO_GROUPS_MAX, refuses them on other jobs, without C, without G, or when C x G x sizeof(apo_group_score) would
 * exceed APO_JOB_CANDIDATE_GROUPS_MAX_BYTES (no overflow); apo_job_prepare allocates the `candidate_groups` output only when
 * the flag is set, apo_job_release frees it; the recordGroupsUpload job checks its buffer and G.
 * With the argument "gpu": the same jobs through a real engine — a recordGroupsUpload job, then resident and host-streaming
 * scoring jobs with the flag return the bytes apo_candidate_groups gives for the same call.
 * Built and run by tests/test_napi_candidate_groups.py. */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "apo_jobs.h"

static int fails;
#define CHECK(cond, ...) do { if (!(cond)) { printf("FAIL: "); printf(__VA_ARGS__); printf("\n"); fails++; } } while (0)

static apo_job scoring(apo_job_kind kind, uint32_t C, uint32_t G, uint32_t flags)
{
	static float dummy[36];
	apo_job j; memset(&j, 0, sizeof j);
	j.kind = kind; j.source = APO_SRC_DIMS; j.C = C; j.G = G; j.K = 1; j.T = 1; j.flags = flags; j.row_bytes = 32;
	j.buf = dummy; j.buf_bytes = (uint64_t)C * 36;
	return j;
}

static void cpu_checks(void)
{
	const uint32_t F = APO_SCORE_CANDIDATE_GROUPS;
	CHECK(sizeof(apo_group_score) == 56, "sizeof(apo_group_score) = %zu", sizeof(apo_group_score));
	CHECK(F == 0x40u && (F & (APO_SCORE_CANDIDATES | APO_SCORE_CANDIDATE_CORPUS | APO_SCORE_CANDIDATE_EXTREMES)) == 0, "flag value");
	const apo_job_kind kinds[4] = {APO_JOB_SCORE_RESIDENT, APO_JOB_SCORE_HOST, APO_JOB_SCORE_HOST_RECORDS, APO_JOB_SCORE_HOST_TUPLES};
	for (int k = 0; k < 4; k++) {
		apo_job a = scoring(kinds[k], 100, 5, F);
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
		CHECK(apo_job_prepare(&a) == APO_OK && a.candidate_groups != NULL && a.candidates == NULL && a.candidate_extremes == NULL,
		      "candidate_groups output not allocated alone (job %d)", k);
		apo_job_release(&a);
		CHECK(a.candidate_groups == NULL, "candidate_groups output not released");
	}
	apo_job b = scoring(APO_JOB_SCORE_RESIDENT, 100, 5, APO_SCORE_CANDIDATE_EXTREMES);
	CHECK(apo_job_validate(&b) == APO_OK && apo_job_prepare(&b) == APO_OK && b.candidate_groups == NULL, "extremes only: groups allocated");
	apo_job_release(&b);
	apo_job g = scoring(APO_JOB_REWARD_BATCH, 4, 5, F);
	g.buf_bytes = 0; g.buf = NULL;
	CHECK(apo_job_validate(&g) == APO_E_ARG && g.err[0], "groups on a non-scoring job accepted");
	apo_job g0 = scoring(APO_JOB_SCORE_RESIDENT, 4, 0, F);
	CHECK(apo_job_validate(&g0) == APO_E_ARG, "G = 0 accepted");
	apo_job g65 = scoring(APO_JOB_SCORE_RESIDENT, 4, 65, F);
	CHECK(apo_job_validate(&g65) == APO_E_ARG, "G = 65 accepted");
	/* the largest C that fits at G = 64, one more, and a C whose byte count overflows 32 bits */
	const uint32_t cmax = (uint32_t)(APO_JOB_CANDIDATE_GROUPS_MAX_BYTES / (64 * sizeof(apo_group_score)));
	apo_job c = scoring(APO_JOB_SCORE_RESIDENT, cmax, 64, F);
	CHECK(apo_job_validate(&c) == APO_OK, "C = %u refused", cmax);
	apo_job c1 = scoring(APO_JOB_SCORE_RESIDENT, cmax + 1, 64, F);
	CHECK(apo_job_validate(&c1) == APO_E_ARG && c1.err[0], "C = %u accepted", cmax + 1);
	apo_job e = scoring(APO_JOB_SCORE_RESIDENT, 0xFFFFFFFFu, 64, F);
	CHECK(apo_job_validate(&e) == APO_E_ARG, "C = 2^32-1 accepted");
	apo_job z = scoring(APO_JOB_SCORE_RESIDENT, 0, 5, F);
	CHECK(apo_job_validate(&z) == APO_E_ARG, "C = 0 with the flag accepted");
	/* recordGroupsUpload: a buffer unless it releases, and 1 <= G <= 64 */
	static uint8_t labels[16];
	apo_job u; memset(&u, 0, sizeof u);
	u.kind = APO_JOB_RECORD_GROUPS_UPLOAD; u.buf = labels; u.buf_bytes = sizeof labels; u.G = 3;
	CHECK(apo_job_validate(&u) == APO_OK, "recordGroupsUpload refused: %s", u.err);
	u.G = 65; u.rc = APO_OK;
	CHECK(apo_job_validate(&u) == APO_E_ARG, "recordGroupsUpload with G = 65 accepted");
	u.G = 0; u.rc = APO_OK;
	CHECK(apo_job_validate(&u) == APO_E_ARG, "recordGroupsUpload with G = 0 accepted");
	u.buf = NULL; u.rc = APO_OK; u.G = 3;
	CHECK(apo_job_validate(&u) == APO_E_ARG, "recordGroupsUpload without a buffer accepted");
	u.buf_bytes = 0; u.rc = APO_OK; u.G = 0;
	CHECK(apo_job_validate(&u) == APO_OK, "releasing the labels refused: %s", u.err);
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
	enum { C = 6, T = 5000, G = 7 };
	float *dims = (float *)malloc(sizeof(float) * C * T * 9);
	unsigned x = 777u;
	for (size_t i = 0; i < (size_t)C * T * 9; i++) {
		x = x * 1103515245u + 12345u;
		const unsigned r = (x >> 8) % 10u;
		dims[i] = r == 0 ? NAN : (r < 4 ? -1.0f : (r < 7 ? 1.0f : 0.5f));
	}
	static uint8_t labels[T];
	for (int t = 0; t < T; t++) labels[t] = (uint8_t)((t / 13) % G);
	apo_job up; memset(&up, 0, sizeof up);
	up.kind = APO_JOB_DIMS_UPLOAD; up.buf = dims; up.buf_bytes = sizeof(float) * C * T * 9; up.C = C; up.T = T;
	CHECK(run(s, &up) == APO_OK, "dimsUpload: %s", up.err);
	apo_job_release(&up);
	apo_job lu; memset(&lu, 0, sizeof lu);
	lu.kind = APO_JOB_RECORD_GROUPS_UPLOAD; lu.buf = labels; lu.buf_bytes = T; lu.G = G;
	CHECK(run(s, &lu) == APO_OK, "recordGroupsUpload: %s", lu.err);

	static apo_group_score direct[C * G];
	apo_job r = scoring(APO_JOB_SCORE_RESIDENT, C, G, APO_SCORE_CANDIDATE_GROUPS);
	r.buf = NULL; r.buf_bytes = 0; r.K = 2;
	CHECK(run(s, &r) == APO_OK && r.candidate_groups, "scoreResident with candidateGroups: %s", r.err);
	CHECK(apo_candidate_groups(s->e, 0, C, G, direct) == APO_OK, "apo_candidate_groups after the job");
	CHECK(r.candidate_groups && memcmp(direct, r.candidate_groups, sizeof direct) == 0, "job groups != apo_candidate_groups");
	for (int c = 0; r.candidate_groups && c < C; c++) {
		uint64_t n = 0;
		for (int g = 0; g < G; g++) n += r.candidate_groups[c * G + g].withReward;
		CHECK(n == r.counts[c], "withReward over the groups != counts[%d]", c);
	}
	apo_job h = scoring(APO_JOB_SCORE_HOST, C, G, APO_SCORE_CANDIDATE_GROUPS | APO_SCORE_CANDIDATE_EXTREMES);
	h.buf = dims; h.buf_bytes = sizeof(float) * C * T * 9; h.T = T; h.K = 2;
	CHECK(run(s, &h) == APO_OK && h.candidate_groups && h.candidate_extremes, "score (host) with candidateGroups: %s", h.err);
	CHECK(h.candidate_groups && memcmp(h.candidate_groups, direct, sizeof direct) == 0, "host-streamed groups != resident");
	apo_job w = scoring(APO_JOB_SCORE_RESIDENT, C, G - 1, APO_SCORE_CANDIDATE_GROUPS);
	w.buf = NULL; w.buf_bytes = 0; w.K = 2;
	CHECK(run(s, &w) == APO_E_ARG, "a job with the wrong G succeeded");
	apo_job n = scoring(APO_JOB_SCORE_RESIDENT, C, 0, 0);
	n.buf = NULL; n.buf_bytes = 0; n.K = 2;
	CHECK(run(s, &n) == APO_OK && n.candidate_groups == NULL, "flag clear: %s", n.err);
	CHECK(apo_candidate_groups(s->e, 0, C, G, direct) == APO_E_STATE, "groups readable after a flag-clear call");
	apo_job_release(&lu); apo_job_release(&r); apo_job_release(&h); apo_job_release(&w); apo_job_release(&n);
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
