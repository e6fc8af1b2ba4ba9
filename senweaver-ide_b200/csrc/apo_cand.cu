// apo_cand.cu — per-candidate breakdown (APO_SCORE_CANDIDATES): the numbers of the corpus report (APO:498-625) answered
// per beam candidate, so that the next beam round can see WHY a candidate scored what it scored.
//
//   k_cand_breakdown<Loader>  one pass over the evaluations a scoring call reads (the same window, candidate offset and
//                             record positions): per candidate the feedback tallies, the exact fixed-point sum and count of
//                             every present dimension over the non-null evaluations, and the first three 'bad' positions.
//                             Domain: a present dimension of a non-null evaluation must satisfy |v| < 2048, where rint(v * 2^52)
//                             still fits in int64; any other value raises P.dom and the call fails with APO_E_ARG (the scoring
//                             kernels bound only finalReward, so d4 = 3000 with w4 = 0 scores normally but has no exact sum)
//   k_cand_report             integers -> apo_candidate_report[C] with the rules of the corpus report (apo_corpus.cuh
//                             report_*), rewardSum / withReward taken from the scoring call's own accumulators
//
// One loader per source family decodes an evaluation to (dims, presence mask, tally) with the decoding of the scoring
// path it mirrors: fp32 rows (Form D), codes + codebook (Form Q, and Form P after k_unpack_p), dictionary entry ->
// codebook / d2book (Form T), records -> reward_dims (Form R / R16).  Validity is the scoring kernels' rule: total weight
// of the presence mask > 0 (LUT), and for records also the VALID flag.
//
// For record sources a second feature (APO_SCORE_CANDIDATE_CORPUS, k_cand_corpus below) goes further: the whole corpus
// report of every candidate's records — patterns, per-mode tallies and tool totals included — by the corpus scan's own code.
#include <cstdlib>
#include "apo_device.cuh"
#include "apo_format.h"
#include "apo_kernels.h"
#include "apo_corpus.cuh"

namespace apo {

constexpr int CB_THREADS = 256;
constexpr int CB_GROUPS = 32;                       // groups of 32 consecutive evaluations per warp tile
constexpr int CB_TILE = 32 * CB_GROUPS;             // evaluations per warp tile (one candidate)
constexpr uint32_t CB_RUN_TILES = 1u << 16;         // flush at least every 64 M evaluations: per-lane counters stay < 2^21
// |v| < 2^11 <=> |rint(v * 2^52)| < 2^63: the dimension values with an exact term.  Every value a loader decodes is an fp32
// widened, and |v| >= 2048, +-inf and NaN are exactly the fp32 magnitudes whose bits are >= 0x45000000 (2048.0f).
constexpr uint32_t CB_FX_BOUND_F32 = 0x45000000u;

// fb: 0 none, 1 good, 2 bad; mag: the largest fp32 magnitude (as bits) of a present dimension, when the loader CHECKs
struct CandEval { double v[APO_NDIM]; uint32_t mask; uint32_t valid; uint32_t fb; uint32_t mag; };

__device__ __forceinline__ uint32_t mag_bits(float f) { return __float_as_uint(f) & 0x7FFFFFFFu; }

// shared tables: the total-weight LUT and the code -> value table of the source (Form Q 8 x 256, Form T 8 x 16)
struct CandSmem { double tw[512]; float tab[8 * 256]; };

// d0 = user_feedback (TCS:677-679): 1 good, -1 bad, anything else (absent included) none
__device__ __forceinline__ uint32_t tally_of_d0(double d0, uint32_t mask) {
	return (mask & 1u) ? (d0 == 1.0 ? 1u : (d0 == -1.0 ? 2u : 0u)) : 0u;
}

// Each loader says whether its values can leave the fixed-point domain (CHECK): record sources cannot (reward_dims yields
// values in [-1, 1] and the duration classes), the fp32 rows and the codebooks can.  MIN_CTAS is the kernel's launch bound
// in CTAs per SM: 2 keeps Form D / Q / W at <= 128 registers (two CTAs per SM) with the check.
struct LoadDims {
	static constexpr int U = 4;                      // groups of 32 evaluations in flight per lane
	static constexpr int MIN_CTAS = 2;
	static constexpr bool CHECK = true;
	struct Raw { float f[APO_NDIM]; };
	__device__ static void fetch(const CandParams &P, uint32_t c, uint64_t t, Raw &R) {
		const float *p = reinterpret_cast<const float *>(P.rows) + ((uint64_t)c * P.pitch_evals + t) * APO_NDIM;
#pragma unroll
		for (int i = 0; i < APO_NDIM; i++) R.f[i] = __ldg(p + i);
	}
	__device__ static void decode(const CandParams &, const CandSmem &S, const Raw &R, CandEval &E) {
		uint32_t mask = 0, mag = 0;
#pragma unroll
		for (int i = 0; i < APO_NDIM; i++) {
			const bool p = R.f[i] == R.f[i];
			E.v[i] = p ? (double)R.f[i] : 0.0;
			mask |= (p ? 1u : 0u) << i;
			mag = max(mag, p ? mag_bits(R.f[i]) : 0u);
		}
		E.mask = mask;
		E.mag = mag;
		E.valid = S.tw[mask] > 0.0 ? 1u : 0u;
		E.fb = tally_of_d0(E.v[0], mask);
	}
};

template <int ROW>
struct LoadRec {
	static constexpr int U = ROW == 32 ? 2 : 4;       // the record decode is a long dependent chain: 4 x 32 B spills
	static constexpr int MIN_CTAS = 1;
	static constexpr bool CHECK = false;
	struct Raw { uint4 q[ROW / 16]; };
	__device__ static void fetch(const CandParams &P, uint32_t c, uint64_t t, Raw &R) {
		const uint4 *p = reinterpret_cast<const uint4 *>(P.rows + ((uint64_t)c * P.pitch_evals + t) * ROW);
#pragma unroll
		for (int k = 0; k < ROW / 16; k++) R.q[k] = __ldg(p + k);
	}
	__device__ static void decode(const CandParams &, const CandSmem &S, const Raw &R, CandEval &E) {
		apo_record r;
		if (ROW == 32) { memcpy(&r, &R, sizeof r); }
		else { apo_record16 p; memcpy(&p, &R, sizeof p); r = unpack16(p); }
		E.mask = reward_dims(r, E.v);                                          // TCS:668-763 in binary64
		E.valid = ((r.flags & APO_F_VALID) && S.tw[E.mask] > 0.0) ? 1u : 0u;  // TCS:606, 784
		E.fb = r.feedback == 1 ? 1u : (r.feedback == 2 ? 2u : 0u);            // as the corpus scan counts (APO:509-516)
	}
};

struct LoadQ {
	static constexpr int U = 4;
	static constexpr int MIN_CTAS = 2;
	static constexpr bool CHECK = true;
	struct Raw { unsigned long long q; float d2; uint32_t li; };
	__device__ static void fetch(const CandParams &P, uint32_t c, uint64_t t, Raw &R) {
		const uint64_t o = (uint64_t)c * P.pitch_evals + t;
		R.q = __ldg(P.q8 + o); R.d2 = __ldg(P.d2 + o); R.li = __ldg(P.li + o);
	}
	__device__ static void decode(const CandParams &, const CandSmem &S, const Raw &R, CandEval &E) {
		uint32_t mask = 0, mag = 0;
#pragma unroll
		for (int j = 0; j < 8; j++) {
			const int dim = j < 2 ? j : j + 1;
			const uint32_t code = (uint32_t)(R.q >> (8 * j)) & 255u;
			const float f = S.tab[256 * j + code];
			E.v[dim] = code == 255u ? 0.0 : (double)f;
			mask |= (code != 255u ? 1u : 0u) << dim;
			mag = max(mag, code == 255u ? 0u : mag_bits(f));
		}
		const bool p2 = ((R.li >> 6) & 1u) != 0;                              // rotated index: dimension 2 lives in bit 6
		E.v[2] = p2 ? (double)R.d2 : 0.0;
		mask |= (p2 ? 1u : 0u) << 2;
		E.mask = mask;
		E.mag = max(mag, p2 ? mag_bits(R.d2) : 0u);
		E.valid = S.tw[mask] > 0.0 ? 1u : 0u;
		E.fb = tally_of_d0(E.v[0], mask);
	}
};

// Form W: one word per evaluation, nibble codes (15 = absent) through the [8][256] fp32 codebook, d2 NaN = absent
struct LoadW {
	static constexpr int U = 4;
	static constexpr int MIN_CTAS = 2;
	static constexpr bool CHECK = true;
	struct Raw { unsigned long long q; };
	__device__ static void fetch(const CandParams &P, uint32_t c, uint64_t t, Raw &R) {
		R.q = __ldg(P.qw + (uint64_t)c * P.pitch_evals + t);
	}
	__device__ static void decode(const CandParams &, const CandSmem &S, const Raw &R, CandEval &E) {
		const uint32_t w = (uint32_t)R.q;
		uint32_t mask = 0, mag = 0;
#pragma unroll
		for (int j = 0; j < 8; j++) {
			const int dim = j < 2 ? j : j + 1;
			const uint32_t nib = (w >> (4 * j)) & 15u;
			const float f = S.tab[256 * j + nib];
			E.v[dim] = nib == 15u ? 0.0 : (double)f;
			mask |= (nib != 15u ? 1u : 0u) << dim;
			mag = max(mag, nib == 15u ? 0u : mag_bits(f));
		}
		const float d2 = __uint_as_float((uint32_t)(R.q >> 32));
		const bool p2 = d2 == d2;
		E.v[2] = p2 ? (double)d2 : 0.0;
		mask |= (p2 ? 1u : 0u) << 2;
		E.mask = mask;
		E.mag = max(mag, p2 ? mag_bits(d2) : 0u);
		E.valid = S.tw[mask] > 0.0 ? 1u : 0u;
		E.fb = tally_of_d0(E.v[0], mask);
	}
};

struct LoadT {
	static constexpr int U = 4;
	static constexpr int MIN_CTAS = 1;
	static constexpr bool CHECK = true;
	struct Raw { uint32_t idx; };
	__device__ static void fetch(const CandParams &P, uint32_t c, uint64_t t, Raw &R) {
		const uint64_t o = (uint64_t)c * P.pitch_evals + t;
		R.idx = (uint32_t)__ldg(P.tl + o) | ((uint32_t)__ldg(P.th + o) << 16);
	}
	__device__ static void decode(const CandParams &P, const CandSmem &S, const Raw &R, CandEval &E) {
		// an index outside the dictionary fails the scoring call (K1t); here it reads as an evaluation with nothing present
		const bool in = R.idx < P.n_tuples;
		const uint32_t w = in ? __ldg(P.tb_pc + R.idx) : 0xFFFFFFFFu;
		const uint32_t k2 = in ? (__ldg(P.tb_pd + R.idx) & 4095u) : 4095u;
		uint32_t mask = 0;
#pragma unroll
		for (int j = 0; j < 8; j++) {
			const int dim = j < 2 ? j : j + 1;
			const uint32_t nib = (w >> (4 * j)) & 15u;
			E.v[dim] = nib == 15u ? 0.0 : (double)S.tab[16 * j + nib];
			mask |= (nib != 15u ? 1u : 0u) << dim;
		}
		const bool p2 = k2 != 4095u;
		E.v[2] = p2 ? (double)__ldg(P.d2book + k2) : 0.0;
		mask |= (p2 ? 1u : 0u) << 2;
		E.mask = mask;
		uint32_t mag = 0;                                                      // every value is an fp32 widened: exact
#pragma unroll
		for (int i = 0; i < APO_NDIM; i++) mag = max(mag, mag_bits((float)E.v[i]));   // absent: 0.0
		E.mag = mag;
		E.valid = S.tw[mask] > 0.0 ? 1u : 0u;
		E.fb = tally_of_d0(E.v[0], mask);
	}
};

// Every warp walks a contiguous range of warp tiles (candidate-major: tile = c * tiles_per_cand + j), keeps its lane
// partials while the candidate stays the same and flushes them into the candidate's words when it changes.  The first
// three 'bad' positions of a run are found with ballots over groups of 32 consecutive evaluations (ascending order
// inside the run), then merged into the candidate's slots with ex_insert, gated on the third slot.
template <class L, int TABLE>
__global__ void __launch_bounds__(CB_THREADS, L::MIN_CTAS)
k_cand_breakdown(const CandParams P, uint32_t tiles_per_cand, uint64_t total_tiles) {
	__shared__ CandSmem S;
	for (int i = threadIdx.x; i < 512; i += CB_THREADS) S.tw[i] = P.lut[i];
	if (TABLE == 1) for (int i = threadIdx.x; i < 8 * 256; i += CB_THREADS) S.tab[i] = P.cbf[i];
	if (TABLE == 2) for (int i = threadIdx.x; i < 8 * 16; i += CB_THREADS) S.tab[i] = P.tbook[i];
	__syncthreads();
	const int lane = threadIdx.x & 31;
	const uint64_t nwarps = (uint64_t)gridDim.x * (CB_THREADS / 32);
	const uint64_t gw = (uint64_t)blockIdx.x * (CB_THREADS / 32) + (threadIdx.x >> 5);
	const uint64_t lo = total_tiles * gw / nwarps, hi = total_tiles * (gw + 1) / nwarps;
	if (lo >= hi) return;

	Acc128 acc[APO_NDIM];
	uint32_t cnt[APO_NDIM], n = 0, good = 0, bad = 0, nfound = 0, run = 0;
	uint32_t dom = 0;                                                    // largest CandEval::mag of a counted evaluation
	unsigned long long f0 = 0ull, f1 = 0ull, f2 = 0ull;                 // first 'bad' positions of the run (nfound of them)
#pragma unroll
	for (int i = 0; i < APO_NDIM; i++) { acc[i].zero(); cnt[i] = 0; }

	auto flush = [&](uint32_t c) {
		long long *w = P.ints + (uint64_t)c * CB_INT;
#pragma unroll
		for (int i = 0; i < APO_NDIM; i++) {
			flush_acc128(acc[i], w + CB_DIM + 4 * i, lane);
			const uint32_t k = warp_sum_u32(cnt[i]);
			if (lane == 0 && k) atomicAdd((unsigned long long *)w + CB_DIM + 4 * i + 3, (unsigned long long)k);
			acc[i].zero(); cnt[i] = 0;
		}
		const uint32_t sn = warp_sum_u32(n), sg = warp_sum_u32(good), sb = warp_sum_u32(bad);
		if (lane == 0) {
			if (sn) atomicAdd((unsigned long long *)w + CB_TALLY, (unsigned long long)sn);
			if (sg) atomicAdd((unsigned long long *)w + CB_TALLY + 1, (unsigned long long)sg);
			if (sb) atomicAdd((unsigned long long *)w + CB_TALLY + 2, (unsigned long long)sb);
			unsigned long long *slots = P.ex + 3ull * c;
			for (uint32_t k = 0; k < nfound; k++) {
				const unsigned long long key = ~(k == 0 ? f0 : (k == 1 ? f1 : f2));   // inverted index (see ex_insert)
				if (key > *((volatile unsigned long long *)&slots[2])) ex_insert(slots, key);
			}
		}
		n = good = bad = 0; nfound = 0; run = 0;
	};

	uint32_t cur = (uint32_t)(lo / tiles_per_cand);
	for (uint64_t tile = lo; tile < hi; tile++) {
		const uint32_t c = (uint32_t)(tile / tiles_per_cand), j = (uint32_t)(tile - (uint64_t)c * tiles_per_cand);
		if (c != cur || run == CB_RUN_TILES) { flush(cur); cur = c; }
		run++;
		const uint64_t t0 = (uint64_t)j * CB_TILE;
		for (int g0 = 0; g0 < CB_GROUPS; g0 += L::U) {
			typename L::Raw R[L::U];
			bool in[L::U];
#pragma unroll
			for (int u = 0; u < L::U; u++) {
				const uint64_t t = t0 + (uint64_t)(g0 + u) * 32 + lane;
				in[u] = t < P.T;
				if (in[u]) L::fetch(P, c, t, R[u]);
			}
#pragma unroll
			for (int u = 0; u < L::U; u++) {
				if (t0 + (uint64_t)(g0 + u) * 32 >= P.T) break;                 // warp-uniform: the rest of the tile is past the row end
				CandEval E;
				bool isbad = false;
				if (in[u]) {
					L::decode(P, S, R[u], E);
					n++;
					good += E.fb == 1u ? 1u : 0u;
					isbad = E.fb == 2u;
					bad += isbad ? 1u : 0u;
					if (E.valid) {
						if (L::CHECK) dom = max(dom, E.mag);
#pragma unroll
						for (int i = 0; i < APO_NDIM; i++) {
							const bool p = (E.mask >> i) & 1u;
							acc[i].add(p ? to_fx(E.v[i]) : 0ll);
							cnt[i] += p ? 1u : 0u;
						}
					}
				}
				if (nfound < 3) {                                                 // warp-uniform
					unsigned int m = __ballot_sync(0xffffffffu, isbad);
					while (m && nfound < 3) {
						const uint32_t pos = (uint32_t)(__ffs((int)m) - 1);
						const unsigned long long gi = P.idx_base + t0 + (uint64_t)(g0 + u) * 32 + pos;
						if (nfound == 0) f0 = gi; else if (nfound == 1) f1 = gi; else f2 = gi;
						nfound++;
						m &= m - 1u;
					}
				}
			}
		}
	}
	flush(cur);
	if (dom >= CB_FX_BOUND_F32) atomicOr(P.dom, 1u);
}

// APO_K1_GRID caps the grids of both per-candidate passes as it caps the scoring kernels' (tuning and tests only, read once)
static uint64_t cand_env_grid() { static const int g = [] { const char *s = getenv("APO_K1_GRID"); return s ? atoi(s) : 0; }(); return g > 0 ? (uint64_t)g : 0; }

template <class L, int TABLE>
static cudaError_t launch_cand(const CandParams &P, int sm_count, cudaStream_t st) {
	const uint32_t tiles_per_cand = (uint32_t)((P.T + CB_TILE - 1) / CB_TILE);
	const uint64_t total_tiles = (uint64_t)tiles_per_cand * P.C;
	if (total_tiles == 0) return cudaSuccess;
	int per_sm = 0;
	cudaError_t err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_cand_breakdown<L, TABLE>, CB_THREADS, 0);
	if (err != cudaSuccess) return err;
	uint64_t grid = (uint64_t)sm_count * (uint64_t)(per_sm > 0 ? per_sm : 1);
	const uint64_t need = (total_tiles + (CB_THREADS / 32) - 1) / (CB_THREADS / 32);
	if (grid > need) grid = need;
	if (cand_env_grid() && cand_env_grid() < grid) grid = cand_env_grid();
	k_cand_breakdown<L, TABLE><<<(unsigned)grid, CB_THREADS, 0, st>>>(P, tiles_per_cand, total_tiles);
	return cudaGetLastError();
}

cudaError_t run_cand_breakdown(const CandParams &P, int source, int sm_count, cudaStream_t st) {
	switch (source) {
	case CAND_DIMS: return launch_cand<LoadDims, 0>(P, sm_count, st);
	case CAND_REC32: return launch_cand<LoadRec<32>, 0>(P, sm_count, st);
	case CAND_REC16: return launch_cand<LoadRec<16>, 0>(P, sm_count, st);
	case CAND_Q: return launch_cand<LoadQ, 1>(P, sm_count, st);
	case CAND_T: return launch_cand<LoadT, 2>(P, sm_count, st);
	case CAND_W: return launch_cand<LoadW, 1>(P, sm_count, st);
	default: return cudaErrorInvalidValue;
	}
}

// one thread per candidate
__global__ void __launch_bounds__(256)
k_cand_report(const long long *ints, const unsigned long long *ex, const long long *partials, uint32_t C, apo_candidate_report *out) {
	const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
	if (c >= C) return;
	const long long *w = ints + (uint64_t)c * CB_INT;
	apo_candidate_report R;
	R.total = (uint64_t)w[CB_TALLY];
	R.good = (uint64_t)w[CB_TALLY + 1];
	R.bad = (uint64_t)w[CB_TALLY + 2];
	R.none = R.total - R.good - R.bad;
	R.goodRate = report_good_rate(R.good, R.bad);                               // APO:546-547
	long long l[4];
#pragma unroll
	for (int q = 0; q < 4; q++) l[q] = partials[(uint64_t)ACC_PER_CAND * c + q];
	R.withReward = (uint64_t)l[3];
	R.rewardSum = limbs_to_double(l);                                           // the limbs score[c] is divided from: same bits
	R.avgReward = report_avg_reward(R.rewardSum, R.withReward);
#pragma unroll 1
	for (int i = 0; i < APO_NDIM; i++) {
		long long d[4];
		for (int q = 0; q < 4; q++) d[q] = w[CB_DIM + 4 * i + q];
		R.dim[i] = report_dimstat(d);
	}
	for (int k = 0; k < 3; k++) {
		const unsigned long long v = ex[3ull * c + k];
		R.badExamples[k] = v == 0ull ? -1ll : (long long)~v;
	}
	out[c] = R;
}

cudaError_t run_cand_report(const long long *ints, const unsigned long long *ex, const long long *partials, uint32_t C,
                            apo_candidate_report *out, cudaStream_t st) {
	if (C == 0) return cudaSuccess;
	k_cand_report<<<(C + 255) / 256, 256, 0, st>>>(ints, ex, partials, C, out);
	return cudaGetLastError();
}

// ================================================================ per-candidate corpus report (APO_SCORE_CANDIDATE_CORPUS)
//   k_cand_corpus<ROW>      the corpus scan (scan_record / scan_flush of apo_corpus.cuh) over the records of every candidate
//                           that a scoring call reads, into one corpus block per candidate
//   k_cand_corpus_report    corpus block -> apo_corpus_report with build_report, the code of the corpus report itself
static_assert(CC_WORDS == CORP_FIXED + APO_NPAT * 3, "one rank's corpus block with its example slots");
constexpr int CC_THREADS = 256;
constexpr int CC_WARPS = CC_THREADS / 32;
constexpr int CC_GROUPS = 32;                               // records per lane in a warp tile (one candidate)
constexpr int CC_TILE = 32 * CC_GROUPS;
constexpr uint32_t CC_RUN_TILES = K2_CHUNK / CC_GROUPS;     // the packed ScanAcc fields hold K2_CHUNK records per lane
static_assert(K2_CHUNK % CC_GROUPS == 0, "a chunk is a whole number of tiles");

// Warps walk candidate-major tiles as k_cand_breakdown does.  A warp flushes its ScanAcc into the candidate's block when the
// candidate changes and after every CC_RUN_TILES tiles; its pattern examples collect in the warp's own 18 shared slots and
// are merged into the candidate's slots at every flush (ex_insert, gated on the third slot).
template <int ROW>
__global__ void __launch_bounds__(CC_THREADS)
k_cand_corpus(const CandCorpusParams P, uint32_t tiles_per_cand, uint64_t total_tiles) {
	__shared__ double s_cat[CAT_WORDS];
	__shared__ double2 s_lut[512];                          // {total weight, reciprocal} per (natural) presence mask
	__shared__ unsigned long long s_ex[CC_WARPS][APO_NPAT * 3];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	if (tid < CAT_WORDS) s_cat[tid] = P.lut[1024 + tid];
	for (int i = tid; i < 512; i += CC_THREADS) s_lut[i] = make_double2(P.lut[i], P.lut[512 + i]);
	if (lane < APO_NPAT * 3) s_ex[warp][lane] = 0ull;
	__syncthreads();
	const uint64_t nwarps = (uint64_t)gridDim.x * CC_WARPS;
	const uint64_t gw = (uint64_t)blockIdx.x * CC_WARPS + warp;
	const uint64_t lo = total_tiles * gw / nwarps, hi = total_tiles * (gw + 1) / nwarps;
	if (lo >= hi) return;
	unsigned long long *ex = s_ex[warp];
	constexpr int U = ROW == 32 ? 2 : 4;                   // records in flight per lane
	ScanAcc A;
	A.zero();
	uint32_t nrec = 0, run = 0;

	auto flush = [&](uint32_t c) {
		long long *corp = P.blk + (uint64_t)c * CC_WORDS;
		scan_flush(A, corp, lane);
		const uint32_t n = warp_sum_u32(nrec);              // CORP_NREC: corpus_tail writes it for the corpus, the pass counts here
		if (lane == 0 && n) atomicAdd((unsigned long long *)corp + CORP_NREC, (unsigned long long)n);
		__syncwarp();
		if (lane < APO_NPAT * 3) {
			const unsigned long long v = ex[lane];
			unsigned long long *slots = (unsigned long long *)corp + CORP_EX + 3 * (lane / 3);
			if (v != 0ull && v > *((volatile unsigned long long *)&slots[2])) ex_insert(slots, v);
			ex[lane] = 0ull;
		}
		__syncwarp();
		A.zero();
		nrec = 0; run = 0;
	};

	uint32_t cur = (uint32_t)(lo / tiles_per_cand);
	for (uint64_t tile = lo; tile < hi; tile++) {
		const uint32_t c = (uint32_t)(tile / tiles_per_cand), j = (uint32_t)(tile - (uint64_t)c * tiles_per_cand);
		if (c != cur || run == CC_RUN_TILES) { flush(cur); cur = c; }
		run++;
		const uint64_t t0 = (uint64_t)j * CC_TILE;
		const uint4 *row = reinterpret_cast<const uint4 *>(P.rows + (uint64_t)c * P.pitch_evals * ROW);
		for (int g0 = 0; g0 < CC_GROUPS; g0 += U) {
			if (t0 + (uint64_t)g0 * 32 >= P.T) break;                           // warp-uniform: the rest of the tile is past the row end
			uint4 q[U][ROW / 16];
#pragma unroll
			for (int u = 0; u < U; u++) {
				const uint64_t t = t0 + (uint64_t)(g0 + u) * 32 + lane;
				if (t < P.T) {
#pragma unroll
					for (int k = 0; k < ROW / 16; k++) q[u][k] = __ldg(row + t * (ROW / 16) + k);
				}
			}
#pragma unroll
			for (int u = 0; u < U; u++) {
				const uint64_t t = t0 + (uint64_t)(g0 + u) * 32 + lane;
				if (t < P.T) {
					apo_record r;
					if constexpr (ROW == 32) { memcpy(&r, q[u], sizeof r); }
					else { apo_record16 p; memcpy(&p, q[u], sizeof p); r = unpack16(p); }
					scan_record<false>(A, r, P.idx_base + t, ex, s_cat, s_lut, P.w2);
					nrec++;
				}
			}
		}
	}
	flush(cur);
}

template <int ROW>
static cudaError_t launch_cand_corpus(const CandCorpusParams &P, int sm_count, cudaStream_t st) {
	const uint32_t tiles_per_cand = (uint32_t)((P.T + CC_TILE - 1) / CC_TILE);
	const uint64_t total_tiles = (uint64_t)tiles_per_cand * P.C;
	if (total_tiles == 0) return cudaSuccess;
	int per_sm = 0;
	cudaError_t err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_cand_corpus<ROW>, CC_THREADS, 0);
	if (err != cudaSuccess) return err;
	uint64_t grid = (uint64_t)sm_count * (uint64_t)(per_sm > 0 ? per_sm : 1);
	const uint64_t need = (total_tiles + CC_WARPS - 1) / CC_WARPS;
	if (grid > need) grid = need;
	if (cand_env_grid() && cand_env_grid() < grid) grid = cand_env_grid();
	k_cand_corpus<ROW><<<(unsigned)grid, CC_THREADS, 0, st>>>(P, tiles_per_cand, total_tiles);
	return cudaGetLastError();
}

cudaError_t run_cand_corpus(const CandCorpusParams &P, int row, int sm_count, cudaStream_t st) {
	if (row == 32) return launch_cand_corpus<32>(P, sm_count, st);
	if (row == 16) return launch_cand_corpus<16>(P, sm_count, st);
	return cudaErrorInvalidValue;
}

// one warp per candidate: the block is copied to the scratch with its example slots as the corpus block holds them (index + 1,
// 0 = none), so that the accumulating block stays intact for later windows of a session; then build_report at one rank.
__global__ void __launch_bounds__(32)
k_cand_corpus_report(const long long *blk, long long *scratch, apo_corpus_report *out) {
	const uint32_t c = blockIdx.x;
	const long long *src = blk + (uint64_t)c * CC_WORDS;
	long long *corp = scratch + (uint64_t)c * CC_WORDS;
	for (int i = threadIdx.x; i < CC_WORDS; i += 32) {
		const long long v = src[i];
		const unsigned long long k = (unsigned long long)v;
		corp[i] = i < CORP_EX ? v : (k == 0ull ? 0ll : (long long)(~k + 1));
	}
	__syncthreads();                                        // build_report reads through L2 what this block wrote (as corpus_tail)
	FinalizeParams F{};
	F.nranks = 1;
	F.report = out + c;
	build_report(F, corp);
}

cudaError_t run_cand_corpus_report(long long *blk, uint32_t C, apo_corpus_report *out, cudaStream_t st) {
	if (C == 0) return cudaSuccess;
	k_cand_corpus_report<<<C, 32, 0, st>>>(blk, blk + (uint64_t)C * CC_WORDS, out);
	return cudaGetLastError();
}

}  // namespace apo
