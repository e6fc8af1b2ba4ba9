/*
 * cand_oracle.h — CPU oracle of the per-candidate breakdown (TEST INFRASTRUCTURE ONLY, see cand_oracle.c).
 * Integers only: sums are exact 128-bit values (lo, hi) of rint(x * 2^52); oracle/candidates.py turns them into the
 * report fields with one rounding each.
 */
#ifndef CAND_ORACLE_H
#define CAND_ORACLE_H
#include <stdint.h>
#include "apo_oracle.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
	uint64_t total, good, bad, none, withReward;
	uint64_t rew_lo; int64_t rew_hi;                       /* sum of rint(finalReward * 2^52) */
	uint64_t dim_lo[ORC_NDIM]; int64_t dim_hi[ORC_NDIM];   /* sum of rint(v * 2^52) over non-null evaluations with dim i present */
	uint64_t dim_count[ORC_NDIM];
	int64_t  badExamples[3];                               /* -1 = none */
	uint32_t refused;                                      /* 1: a counted present dimension with |v| >= 2048 (term left out) */
	uint32_t pad;
} orc_cand_fx;

/* Form D [C][pitch][9] fp32 (NaN = absent); positions idx_base + t */
void orc_cand_dims(const float *dims, uint32_t C, uint64_t T, uint64_t pitch_evals, uint64_t idx_base, const double w[ORC_NDIM],
                   orc_cand_fx *out);
/* Form R [C][pitch] */
void orc_cand_records(const orc_record *recs, uint32_t C, uint64_t T, uint64_t pitch, uint64_t idx_base, const double w[ORC_NDIM],
                      orc_cand_fx *out);
/* the listed candidates over generated Form D evaluations [t0, t0+T) (never materialised); threads over record slices,
 * merged in slice order: any thread count gives the same result */
void orc_cand_generated(uint64_t seed, const uint32_t *cands, uint32_t ncand, uint64_t t0, uint64_t T, uint32_t agent_permille,
                        const double w[ORC_NDIM], orc_cand_fx *out, int nthreads);
/* the same over the generator's rollout records (Form R; Form R16 packs them without changing any output) */
void orc_cand_generated_records(uint64_t seed, const uint32_t *cands, uint32_t ncand, uint64_t t0, uint64_t T, uint32_t agent_permille,
                                const double w[ORC_NDIM], orc_cand_fx *out, int nthreads);

#ifdef __cplusplus
}
#endif
#endif
