#define _POSIX_C_SOURCE 199309L
/* The dimsTuples job in the addon's job core (napi/apo_jobs.c): validation accepts cap <= APO_TUPLES_MAX and refuses
 * anything above it; the job takes its turn in the handle's FIFO between other jobs, also when it fails (on a handle without
 * an engine it fails with APO_E_STATE in its turn, it does not fall back).
 * With the argument "gpu": through a real engine it refuses before a load, builds Form T after one (n_out = nTuples, equal to
 * apo_dims_tuples on a second engine), and a cap below the distinct count fails with APO_E_STATE and an error text.
 * Built and run by tests/test_napi_tuples.py. */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include "apo_jobs.h"

static int fails;
#define CHECK(cond, ...) do { if (!(cond)) { printf("FAIL: "); printf(__VA_ARGS__); printf("\n"); fails++; } } while (0)

#define NJOBS 60
static apo_serial *S;
static apo_job jobs[NJOBS];
static int order[NJOBS], norder, next_job;

static void hook(void *arg) { order[norder++] = (int)(intptr_t)arg; }

static void *worker(void *p)
{
	(void)p;
	for (;;) {
		const int i = __atomic_fetch_add(&next_job, 1, __ATOMIC_SEQ_CST);
		if (i >= NJOBS) break;
		if (i % 3 == 0) { struct timespec ts = {0, 50000}; nanosleep(&ts, NULL); }
		apo_job_run(S, &jobs[i]);
	}
	return NULL;
}

static apo_job tuples_job(uint32_t cap)
{
	apo_job j; memset(&j, 0, sizeof j);
	j.kind = APO_JOB_DIMS_TUPLES; j.cap = cap;
	return j;
}

static void cpu_checks(void)
{
	apo_job a = tuples_job(APO_TUPLES_MAX);
	CHECK(apo_job_validate(&a) == APO_OK, "cap = APO_TUPLES_MAX refused: %s", a.err);
	apo_job b = tuples_job(0);
	CHECK(apo_job_validate(&b) == APO_OK, "cap = 0 refused: %s", b.err);
	apo_job c = tuples_job(APO_TUPLES_MAX + 1);
	CHECK(apo_job_validate(&c) == APO_E_ARG && c.err[0], "cap = APO_TUPLES_MAX + 1 accepted");
	apo_job d = tuples_job(0xFFFFFFFFu);
	CHECK(apo_job_validate(&d) == APO_E_ARG, "cap = 2^32 - 1 accepted");

	/* FIFO: hooks around dimsTuples jobs (valid ones fail in their turn without an engine, invalid ones before) */
	S = apo_serial_create_detached();
	for (int i = 0; i < NJOBS; i++) {
		memset(&jobs[i], 0, sizeof jobs[i]);
		if (i % 10 == 4) jobs[i] = tuples_job(i % 20 == 4 ? 1000u : APO_TUPLES_MAX + 1);
		else { jobs[i].kind = APO_JOB_TEST_HOOK; jobs[i].hook = hook; jobs[i].hook_arg = (void *)(intptr_t)i; }
		apo_job_validate(&jobs[i]);
		jobs[i].ticket = apo_serial_ticket(S);
	}
	pthread_t th[6];
	for (int i = 0; i < 6; i++) pthread_create(&th[i], NULL, worker, NULL);
	for (int i = 0; i < 6; i++) pthread_join(th[i], NULL);
	int want = 0, pos = 0;
	for (; want < NJOBS; want++) {
		if (want % 10 == 4) continue;
		if (pos >= norder || order[pos] != want) { CHECK(0, "position %d ran job %d, expected %d", pos, pos < norder ? order[pos] : -1, want); break; }
		pos++;
	}
	CHECK(norder == NJOBS - NJOBS / 10, "%d hooks ran", norder);
	for (int i = 4; i < NJOBS; i += 10) {
		const int expect = i % 20 == 4 ? APO_E_STATE : APO_E_ARG;
		CHECK(jobs[i].rc == expect && jobs[i].err[0], "dimsTuples job %d rc=%d, expected %d", i, jobs[i].rc, expect);
	}
	apo_serial_destroy(S);
}

static void gpu_checks(void)
{
	char err[256];
	apo_serial *s = apo_serial_create(0, err, sizeof err);
	CHECK(s != NULL, "no engine: %s", err);
	if (!s) return;
	apo_job j = tuples_job(APO_TUPLES_MAX);
	apo_job_validate(&j); j.ticket = apo_serial_ticket(s); apo_job_run(s, &j);
	CHECK(j.rc == APO_E_STATE && j.err[0], "dimsTuples before a load: rc=%d", j.rc);
	CHECK(apo_dims_generate(s->e, 77, 0, 5, 0, 20011, 300) == APO_OK, "apo_dims_generate failed");
	apo_job k = tuples_job(APO_TUPLES_MAX);
	apo_job_validate(&k); k.ticket = apo_serial_ticket(s); apo_job_run(s, &k);
	CHECK(k.rc == APO_OK && k.n_out > 0, "dimsTuples after a load: rc=%d (%s)", k.rc, k.err);
	apo_engine *e2 = NULL;
	uint32_t n2 = 0;
	CHECK(apo_create(0, &e2) == APO_OK && apo_dims_generate(e2, 77, 0, 5, 0, 20011, 300) == APO_OK && apo_dims_tuples(e2, APO_TUPLES_MAX, &n2) == APO_OK,
	      "second engine");
	CHECK(n2 == k.n_out, "job n_out %llu != apo_dims_tuples %u", (unsigned long long)k.n_out, n2);
	apo_destroy(e2);
	apo_job m = tuples_job(n2 - 1);
	apo_job_validate(&m); m.ticket = apo_serial_ticket(s); apo_job_run(s, &m);
	CHECK(m.rc == APO_E_STATE && m.err[0], "cap below the distinct count: rc=%d", m.rc);
	apo_serial_destroy(s);
}

int main(int argc, char **argv)
{
	cpu_checks();
	if (argc > 1 && strcmp(argv[1], "gpu") == 0) gpu_checks();
	if (fails) return 1;
	printf("OK\n");
	return 0;
}
