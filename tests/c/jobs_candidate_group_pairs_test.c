/* The paired comparisons per record group in the addon's job core (napi/apo_jobs.c): validation accepts them on every scoring
 * job, refuses them on other jobs, without C, without G (or G above APO_GROUPS_MAX), or when C x G x sizeof(struct
 * apo_candidate_pair) would exceed APO_JOB_CANDIDATE_GROUP_PAIRS_MAX_BYTES (no overflow); apo_job_prepare allocates the
 * `candidate_group_pairs` output ([C][G]) only when the flag is set, apo_job_release frees it.
 * With the argument "gpu": the same jobs through a real engine — labels and refs upload jobs, then resident and
 * host-streaming scoring jobs with the flag return the bytes apo_candidate_group_pairs gives for the same call, and summed over
 * the labels every integer field is apo_candidate_pairs'.
 * Built and run by tests/test_napi_candidate_group_pairs.py. */
#include <math.h>
#include <stddef.h>
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
	const uint32_t F = APO_SCORE_CANDIDATE_GROUP_PAIRS;
	CHECK(F == 0x200u && (F & (APO_SCORE_CANDIDATES | APO_SCORE_CANDIDATE_CORPUS | APO_SCORE_CANDIDATE_EXTREMES | APO_SCORE_CANDIDATE_GROUPS |
	                           APO_SCORE_CANDIDATE_SPREAD | APO_SCORE_CANDIDATE_PAIRS)) == 0, "flag value");
	const apo_job_kind kinds[4] = {APO_JOB_SCORE_RESIDENT, APO_JOB_SCORE_HOST, APO_JOB_SCORE_HOST_RECORDS, APO_JOB_SCORE_HOST_TUPLES};
	for (int k = 0; k < 4; k++) {
		apo_job a = scoring(kinds[k], 100, 7, F);
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
		CHECK(apo_job_prepare(&a) == APO_OK && a.candidate_group_pairs != NULL && a.candidate_pairs == NULL && a.candidate_groups == NULL &&
		      a.candidates == NULL, "candidate_group_pairs output not allocated alone (job %d)", k);
		if (a.candidate_group_pairs) memset(a.candidate_group_pairs, 0, sizeof(struct apo_candidate_pair) * 100 * 7);   /* [C][G] */
		apo_job_release(&a);
		CHECK(a.candidate_group_pairs == NULL, "candidate_group_pairs output not released");
	}
	apo_job b = scoring(APO_JOB_SCORE_RESIDENT, 100, 7, APO_SCORE_CANDIDATE_PAIRS | APO_SCORE_CANDIDATE_GROUPS);
	CHECK(apo_job_validate(&b) == APO_OK && apo_job_prepare(&b) == APO_OK && b.candidate_group_pairs == NULL, "pairs + groups: group pairs allocated");
	apo_job_release(&b);
	apo_job g = scoring(APO_JOB_REWARD_BATCH, 4, 2, F);
	g.buf_bytes = 0; g.buf = NULL;
	CHECK(apo_job_validate(&g) == APO_E_ARG && g.err[0], "group pairs on a non-scoring job accepted");
	apo_job g0 = scoring(APO_JOB_SCORE_RESIDENT, 4, 0, F);
	CHECK(apo_job_validate(&g0) == APO_E_ARG && g0.err[0], "G = 0 with the flag accepted");
	apo_job g65 = scoring(APO_JOB_SCORE_RESIDENT, 4, APO_GROUPS_MAX + 1, F);
	CHECK(apo_job_validate(&g65) == APO_E_ARG, "G = 65 accepted");
	apo_job z = scoring(APO_JOB_SCORE_RESIDENT, 0, 2, F);
	CHECK(apo_job_validate(&z) == APO_E_ARG, "C = 0 with the flag accepted");
	/* the largest C that fits at G = 64, one more, and a C whose byte count passes 32 bits */
	const uint32_t cmax = (uint32_t)(APO_JOB_CANDIDATE_GROUP_PAIRS_MAX_BYTES / (64 * sizeof(struct apo_candidate_pair)));
	apo_job c = scoring(APO_JOB_SCORE_RESIDENT, cmax, 64, F);
	CHECK(apo_job_validate(&c) == APO_OK, "C = %u at G = 64 refused", cmax);
	apo_job c1 = scoring(APO_JOB_SCORE_RESIDENT, cmax + 1, 64, F);
	CHECK(apo_job_validate(&c1) == APO_E_ARG && c1.err[0], "C = %u at G = 64 accepted", cmax + 1);
	apo_job e = scoring(APO_JOB_SCORE_RESIDENT, 0xFFFFFFFFu, 64, F);
	CHECK(apo_job_validate(&e) == APO_E_ARG, "C = 2^32-1 accepted");
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
	enum { C = 6, T = 5000, G = 5 };
	float *dims = (float *)malloc(sizeof(float) * C * T * 9);
	unsigned x = 1993u;
	for (size_t i = 0; i < (size_t)C * T * 9; i++) {
		x = x * 1103515245u + 12345u;
		const unsigned r = (x >> 8) % 10u;
		dims[i] = r == 0 ? NAN : (r < 4 ? -1.0f : (r < 7 ? 1.0f : 0.5f));
	}
	apo_job up; memset(&up, 0, sizeof up);
	up.kind = APO_JOB_DIMS_UPLOAD; up.buf = dims; up.buf_bytes = sizeof(float) * C * T * 9; up.C = C; up.T = T;
	CHECK(run(s, &up) == APO_OK, "dimsUpload: %s", up.err);
	apo_job_release(&up);
	static uint8_t labels[T];
	for (int t = 0; t < T; t++) labels[t] = (uint8_t)(t % G);
	apo_job lu; memset(&lu, 0, sizeof lu);
	lu.kind = APO_JOB_RECORD_GROUPS_UPLOAD; lu.buf = labels; lu.buf_bytes = T; lu.G = G;
	CHECK(run(s, &lu) == APO_OK, "recordGroupsUpload: %s", lu.err);
	uint32_t refs[C] = {APO_PAIR_NONE, 0, 0, 4, 5, 5};
	apo_job u; memset(&u, 0, sizeof u);
	u.kind = APO_JOB_CANDIDATE_REFS_UPLOAD; u.buf = refs; u.buf_bytes = sizeof refs; u.C = C;
	CHECK(run(s, &u) == APO_OK, "candidateRefsUpload: %s", u.err);

	static struct apo_candidate_pair direct[C * G], pairs[C];
	apo_job r = scoring(APO_JOB_SCORE_RESIDENT, C, G, APO_SCORE_CANDIDATE_GROUP_PAIRS | APO_SCORE_CANDIDATE_PAIRS);
	r.buf = NULL; r.buf_bytes = 0; r.K = 2;
	CHECK(run(s, &r) == APO_OK && r.candidate_group_pairs && r.candidate_pairs, "scoreResident with candidateGroupPairs: %s", r.err);
	CHECK(apo_candidate_group_pairs(s->e, 0, C, G, direct) == APO_OK, "apo_candidate_group_pairs after the job");
	CHECK(apo_candidate_pairs(s->e, 0, C, pairs) == APO_OK, "apo_candidate_pairs after the job");
	CHECK(r.candidate_group_pairs && memcmp(direct, r.candidate_group_pairs, sizeof direct) == 0, "job group pairs != apo_candidate_group_pairs");
	for (int c = 0; c < C; c++) {
		uint64_t n = 0, w = 0, l = 0, ti = 0, co = 0, ro = 0, lo = 0, hi = 0, carry;
		for (int g = 0; g < G; g++) {
			const struct apo_candidate_pair *p = &direct[c * G + g];
			CHECK(p->ref == refs[c], "ref of (%d, %d)", c, g);
			if (refs[c] == APO_PAIR_NONE) CHECK(p->n == 0 && isnan(p->meanDiff), "(%d, %d) without a reference", c, g);
			n += p->n; w += p->wins; l += p->losses; ti += p->ties; co += p->candOnly; ro += p->refOnly;
			carry = lo + p->sumLo < lo; lo += p->sumLo; hi += (uint64_t)p->sumHi + carry;
		}
		CHECK(n == pairs[c].n && w == pairs[c].wins && l == pairs[c].losses && ti == pairs[c].ties && co == pairs[c].candOnly &&
		      ro == pairs[c].refOnly, "tallies of %d summed over the labels", c);
		CHECK(lo == pairs[c].sumLo && hi == (uint64_t)pairs[c].sumHi, "D1 of %d summed over the labels", c);
	}
	apo_job h = scoring(APO_JOB_SCORE_HOST, C, G, APO_SCORE_CANDIDATE_GROUP_PAIRS | APO_SCORE_CANDIDATE_SPREAD);
	h.buf = dims; h.buf_bytes = sizeof(float) * C * T * 9; h.T = T; h.K = 2;
	CHECK(run(s, &h) == APO_OK && h.candidate_group_pairs && h.candidate_spread && !h.candidate_groups,
	      "score (host) with candidateGroupPairs: %s", h.err);
	CHECK(h.candidate_group_pairs && memcmp(h.candidate_group_pairs, direct, sizeof direct) == 0, "host-streamed group pairs != resident");
	apo_job n = scoring(APO_JOB_SCORE_RESIDENT, C, 0, 0);
	n.buf = NULL; n.buf_bytes = 0; n.K = 2;
	CHECK(run(s, &n) == APO_OK && n.candidate_group_pairs == NULL, "flag clear: %s", n.err);
	CHECK(apo_candidate_group_pairs(s->e, 0, C, G, direct) == APO_E_STATE, "group pairs readable after a flag-clear call");
	apo_job rel; memset(&rel, 0, sizeof rel);
	rel.kind = APO_JOB_CANDIDATE_REFS_UPLOAD; rel.C = 0;
	CHECK(run(s, &rel) == APO_OK, "refs release: %s", rel.err);
	apo_job q = scoring(APO_JOB_SCORE_RESIDENT, C, G, APO_SCORE_CANDIDATE_GROUP_PAIRS);
	q.buf = NULL; q.buf_bytes = 0; q.K = 2;
	CHECK(run(s, &q) == APO_E_STATE, "group pairs without refs accepted");
	apo_job_release(&lu); apo_job_release(&u); apo_job_release(&r); apo_job_release(&h); apo_job_release(&n); apo_job_release(&rel);
	apo_job_release(&q);
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
