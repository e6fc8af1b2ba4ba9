// apo_cand.cu — per-candidate breakdown (APO_SCORE_CANDIDATES): the numbers of the corpus report (APO:498-625) answered
// per beam candidate, so that the next beam round can see WHY a candidate scored what it scored.
//
//   k_cand_breakdown<Loader>  one pass over the evaluations a scoring call reads (the same window, candidate offset and
//                             record positions): per candidate the feedback tallies, the exact fixed-point sum and count of
//                             every present dimension over the non-null evaluations, and the first three 'bad' positions.
//                             Domain: a present dimension of a non-null evaluation must satisfy |v| < 2048, where rint(v * 2^52)
//                             still fits in int64; any other value raises CandParams::dom and the call fails with APO_E_ARG (the
//                             scoring kernels bound only finalReward, so d4 = 3000 with w4 = 0 scores normally but has no exact sum)
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
// The extremes, the group scores, the reward spread, the paired comparison and its split by record group follow.  Every pass
// is one walk (cand_walk) over the same warp tiles with its own per-evaluation step and flush, and one launcher sizes every
// walk's grid (walk_grid).
#include <atomic>
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

// The finalReward of a non-null evaluation, bit for bit the one the scoring kernels sum: TCS:777-784 in push order with
// absent values +0.0, divided through the total-weight LUT (tw) and its reciprocals (rc) as div_lut does
template <bool RECIP>
__device__ __forceinline__ double cand_final_reward(const CandEval &E, const Weights &W, const double *tw, const double *rc) {
	double ws = 0.0;
#pragma unroll
	for (int i = 0; i < APO_NDIM; i++) ws = __dadd_rn(ws, __dmul_rn(E.v[i], W.w[i]));
	return div_lut<RECIP>(ws, make_double2(tw[E.mask], rc[E.mask]));
}

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
	__device__ static void fetch(const CandEvals &P, uint32_t c, uint64_t t, Raw &R) {
		const float *p = reinterpret_cast<const float *>(P.rows) + ((uint64_t)c * P.pitch_evals + t) * APO_NDIM;
#pragma unroll
		for (int i = 0; i < APO_NDIM; i++) R.f[i] = __ldg(p + i);
	}
	__device__ static void decode(const CandEvals &, const CandSmem &S, const Raw &R, CandEval &E) {
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
	__device__ static void fetch(const CandEvals &P, uint32_t c, uint64_t t, Raw &R) {
		const uint4 *p = reinterpret_cast<const uint4 *>(P.rows + ((uint64_t)c * P.pitch_evals + t) * ROW);
#pragma unroll
		for (int k = 0; k < ROW / 16; k++) R.q[k] = __ldg(p + k);
	}
	__device__ static apo_record record(const Raw &R) {
		apo_record r;
		if constexpr (ROW == 32) { memcpy(&r, &R, sizeof r); }
		else { apo_record16 p; memcpy(&p, &R, sizeof p); r = unpack16(p); }
		return r;
	}
	__device__ static void decode(const CandEvals &, const CandSmem &S, const Raw &R, CandEval &E) {
		const apo_record r = record(R);
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
	__device__ static void fetch(const CandEvals &P, uint32_t c, uint64_t t, Raw &R) {
		const uint64_t o = (uint64_t)c * P.pitch_evals + t;
		R.q = __ldg(P.q8 + o); R.d2 = __ldg(P.d2 + o); R.li = __ldg(P.li + o);
	}
	__device__ static void decode(const CandEvals &, const CandSmem &S, const Raw &R, CandEval &E) {
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
	__device__ static void fetch(const CandEvals &P, uint32_t c, uint64_t t, Raw &R) {
		R.q = __ldg(P.qw + (uint64_t)c * P.pitch_evals + t);
	}
	__device__ static void decode(const CandEvals &, const CandSmem &S, const Raw &R, CandEval &E) {
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
	__device__ static void fetch(const CandEvals &P, uint32_t c, uint64_t t, Raw &R) {
		const uint64_t o = (uint64_t)c * P.pitch_evals + t;
		R.idx = (uint32_t)__ldg(P.tl + o) | ((uint32_t)__ldg(P.th + o) << 16);
	}
	__device__ static void decode(const CandEvals &P, const CandSmem &S, const Raw &R, CandEval &E) {
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

// ================================================================ the walk every per-candidate pass shares
constexpr int CB_WARPS = CB_THREADS / 32;

// the total-weight LUT, its reciprocals into rc for the passes that divide as div_lut does (DIV), and the source's
// code -> value table
template <int TABLE, bool DIV = false>
__device__ __forceinline__ void stage_tables(const CandEvals &P, CandSmem &S, double *rc = nullptr) {
	for (int i = threadIdx.x; i < 512; i += CB_THREADS) {
		S.tw[i] = P.lut[i];
		if (DIV) rc[i] = P.lut[512 + i];
	}
	if (TABLE == 1) for (int i = threadIdx.x; i < 8 * 256; i += CB_THREADS) S.tab[i] = P.cbf[i];
	if (TABLE == 2) for (int i = threadIdx.x; i < 8 * 16; i += CB_THREADS) S.tab[i] = P.tbook[i];
	__syncthreads();
}

__device__ __forceinline__ uint64_t cand_warp() { return (uint64_t)blockIdx.x * CB_WARPS + (threadIdx.x >> 5); }

struct NoSide { __device__ uint32_t operator()(uint64_t) const { return 0u; } };
// the second row a pass reads per candidate: none (every pass but the paired comparison); U: groups of 32 evaluations a lane
// keeps in flight over loader L
struct NoPair {
	static constexpr bool PAIR = false;
	template <class L> static constexpr int U = L::U;
	__device__ uint32_t operator()(uint32_t) const { return 0u; }
};

// Warp tiles of CB_TILE evaluations run candidate-major (tile = c * tiles_per_cand + j), and every warp walks a contiguous
// range of them (the range k_cand_extremes_merge inverts).  A lane keeps U = Pair::U<L> groups of 32 evaluations in flight, then
// each(c, t, in, R, s) sees them in order: t is the lane's evaluation, in says whether it lies inside the row, and only then
// do R (its fetch) and s (side(t), fetched with it) hold anything.  A group wholly past the row end ends the tile,
// warp-uniformly.  flush(c) ends the warp's run of candidate c: when the candidate changes, after every RUN tiles (0: never)
// and after the last tile.  A pass with a second row (Pair::PAIR) names it per candidate, pair(c) (APO_PAIR_NONE: the
// candidate's tiles are skipped, warp-uniformly, and nothing of them is loaded); that row's evaluation t is fetched in the same
// in-flight group as the candidate's own, and each(c, t, in, R, Q, s) sees it as Q.
template <class L, uint32_t RUN, class Each, class Flush, class Side = NoSide, class Pair = NoPair>
__device__ __forceinline__ void cand_walk(const CandEvals &P, uint32_t tiles_per_cand, uint64_t total_tiles, Each &&each, Flush &&flush,
                                          Side side = {}, Pair pair = {}) {
	constexpr int U = Pair::template U<L>;
	const int lane = threadIdx.x & 31;
	const uint64_t nwarps = (uint64_t)gridDim.x * CB_WARPS, gw = cand_warp();
	const uint64_t lo = total_tiles * gw / nwarps, hi = total_tiles * (gw + 1) / nwarps;
	if (lo >= hi) return;
	uint32_t cur = (uint32_t)(lo / tiles_per_cand), run = 0;
	for (uint64_t tile = lo; tile < hi; tile++) {
		const uint32_t c = (uint32_t)(tile / tiles_per_cand), j = (uint32_t)(tile - (uint64_t)c * tiles_per_cand);
		if (c != cur || (RUN && run == RUN)) { flush(cur); cur = c; run = 0; }
		run++;
		uint32_t rc = 0;
		if constexpr (Pair::PAIR) {
			rc = pair(c);
			if (rc == APO_PAIR_NONE) continue;                              // warp-uniform: c is the warp's candidate
		}
		const uint64_t t0 = (uint64_t)j * CB_TILE;
		for (int g0 = 0; g0 < CB_GROUPS; g0 += U) {
			typename L::Raw R[U], Q[Pair::PAIR ? U : 1];
			bool in[U];
			uint32_t s[U];
#pragma unroll
			for (int u = 0; u < U; u++) {
				const uint64_t t = t0 + (uint64_t)(g0 + u) * 32 + lane;
				in[u] = t < P.T;
				s[u] = in[u] ? side(t) : 0u;
				if (in[u]) {
					L::fetch(P, c, t, R[u]);
					if constexpr (Pair::PAIR) L::fetch(P, rc, t, Q[u]);
				}
			}
#pragma unroll
			for (int u = 0; u < U; u++) {
				const uint64_t t = t0 + (uint64_t)(g0 + u) * 32 + lane;
				if (t - lane >= P.T) break;                                 // warp-uniform: the rest of the tile is past the row end
				if constexpr (Pair::PAIR) each(c, t, in[u], R[u], Q[u], s[u]);
				else each(c, t, in[u], R[u], s[u]);
			}
		}
	}
	flush(cur);
}

// APO_K1_GRID caps the grids of the per-candidate passes as it caps the scoring kernels' (tuning and tests only, read once)
static uint64_t cand_env_grid() { static const int g = [] { const char *s = getenv("APO_K1_GRID"); return s ? atoi(s) : 0; }(); return g > 0 ? (uint64_t)g : 0; }

// The tiles of a launch over P and the grid of a walk kernel for them: as many CTAs as the SMs hold at once (with smem bytes
// of dynamic shared memory each), no more than the tiles need, at most APO_K1_GRID.  grid = 0: nothing to walk.
struct Walk { uint32_t tiles_per_cand; uint64_t total_tiles, grid; };

template <class K>
static cudaError_t walk_grid(K *kernel, const CandEvals &P, int sm_count, Walk &w, size_t smem = 0) {
	w.tiles_per_cand = (uint32_t)((P.T + CB_TILE - 1) / CB_TILE);
	w.total_tiles = (uint64_t)w.tiles_per_cand * P.C;
	w.grid = 0;
	if (w.total_tiles == 0) return cudaSuccess;
	int per_sm = 0;
	const cudaError_t err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, CB_THREADS, smem);
	if (err != cudaSuccess) return err;
	w.grid = (uint64_t)sm_count * (uint64_t)(per_sm > 0 ? per_sm : 1);
	const uint64_t need = (w.total_tiles + CB_WARPS - 1) / CB_WARPS;
	if (w.grid > need) w.grid = need;
	if (cand_env_grid() && cand_env_grid() < w.grid) w.grid = cand_env_grid();
	return cudaSuccess;
}

// a pass that is its walk kernel alone
template <class X>
static cudaError_t launch_walk(void (*kernel)(X, uint32_t, uint64_t), const X &x, int sm_count, cudaStream_t st, size_t smem = 0) {
	Walk w;
	const cudaError_t err = walk_grid(kernel, x.src, sm_count, w, smem);
	if (err != cudaSuccess || w.grid == 0) return err;
	kernel<<<(unsigned)w.grid, CB_THREADS, smem, st>>>(x, w.tiles_per_cand, w.total_tiles);
	return cudaGetLastError();
}

// ================================================================ per-candidate breakdown (APO_SCORE_CANDIDATES)
// Every warp keeps its lane partials while the candidate stays the same and flushes them into the candidate's words.  The
// first three 'bad' positions of a run are found with ballots over groups of 32 consecutive evaluations (ascending order
// inside the run), then merged into the candidate's slots with ex_insert, gated on the third slot.
template <class L, int TABLE>
__global__ void __launch_bounds__(CB_THREADS, L::MIN_CTAS)
k_cand_breakdown(const CandParams X, uint32_t tiles_per_cand, uint64_t total_tiles) {
	const CandEvals &P = X.src;
	__shared__ CandSmem S;
	stage_tables<TABLE>(P, S);
	const int lane = threadIdx.x & 31;
	Acc128 acc[APO_NDIM];
	uint32_t cnt[APO_NDIM], n = 0, good = 0, bad = 0, nfound = 0;
	uint32_t dom = 0;                                                    // largest CandEval::mag of a counted evaluation
	unsigned long long f0 = 0ull, f1 = 0ull, f2 = 0ull;                 // first 'bad' positions of the run (nfound of them)
#pragma unroll
	for (int i = 0; i < APO_NDIM; i++) { acc[i].zero(); cnt[i] = 0; }

	auto flush = [&](uint32_t c) {
		long long *w = X.ints + (uint64_t)c * CB_INT;
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
			unsigned long long *slots = X.ex + 3ull * c;
			for (uint32_t k = 0; k < nfound; k++) {
				const unsigned long long key = ~(k == 0 ? f0 : (k == 1 ? f1 : f2));   // inverted index (see ex_insert)
				if (key > *((volatile unsigned long long *)&slots[2])) ex_insert(slots, key);
			}
		}
		n = good = bad = 0; nfound = 0;
	};
	auto each = [&](uint32_t, uint64_t t, bool in, const typename L::Raw &R, uint32_t) {
		bool isbad = false;
		if (in) {
			CandEval E;
			L::decode(P, S, R, E);
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
		if (nfound < 3) {                                                     // warp-uniform
			unsigned int m = __ballot_sync(0xffffffffu, isbad);
			while (m && nfound < 3) {
				const uint32_t pos = (uint32_t)(__ffs((int)m) - 1);
				const unsigned long long gi = P.idx_base + (t - lane) + pos;
				if (nfound == 0) f0 = gi; else if (nfound == 1) f1 = gi; else f2 = gi;
				nfound++;
				m &= m - 1u;
			}
		}
	};
	cand_walk<L, CB_RUN_TILES>(P, tiles_per_cand, total_tiles, each, flush);
	if (dom >= CB_FX_BOUND_F32) atomicOr(X.dom, 1u);
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
constexpr uint32_t CC_RUN_TILES = K2_CHUNK / CB_GROUPS;     // the packed ScanAcc fields hold K2_CHUNK records per lane
static_assert(K2_CHUNK % CB_GROUPS == 0, "a chunk is a whole number of tiles");

// The walk of the breakdown over LoadRec's records.  A warp flushes its ScanAcc into the candidate's block when the candidate
// changes and after every CC_RUN_TILES tiles; its pattern examples collect in the warp's own 18 shared slots and are merged
// into the candidate's slots at every flush (ex_insert, gated on the third slot).
template <int ROW>
__global__ void __launch_bounds__(CB_THREADS)
k_cand_corpus(const CandCorpusParams X, uint32_t tiles_per_cand, uint64_t total_tiles) {
	const CandEvals &P = X.src;
	__shared__ double s_cat[CAT_WORDS];
	__shared__ double2 s_lut[512];                          // {total weight, reciprocal} per (natural) presence mask
	__shared__ unsigned long long s_ex[CB_WARPS][APO_NPAT * 3];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	if (tid < CAT_WORDS) s_cat[tid] = P.lut[1024 + tid];
	for (int i = tid; i < 512; i += CB_THREADS) s_lut[i] = make_double2(P.lut[i], P.lut[512 + i]);
	if (lane < APO_NPAT * 3) s_ex[warp][lane] = 0ull;
	__syncthreads();
	unsigned long long *ex = s_ex[warp];
	ScanAcc A;
	A.zero();
	uint32_t nrec = 0;

	auto flush = [&](uint32_t c) {
		long long *corp = X.blk + (uint64_t)c * CC_WORDS;
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
		nrec = 0;
	};
	auto each = [&](uint32_t, uint64_t t, bool in, const typename LoadRec<ROW>::Raw &R, uint32_t) {
		if (!in) return;
		scan_record<false>(A, LoadRec<ROW>::record(R), P.idx_base + t, ex, s_cat, s_lut, X.w2);
		nrec++;
	};
	cand_walk<LoadRec<ROW>, CC_RUN_TILES>(P, tiles_per_cand, total_tiles, each, flush);
}

cudaError_t run_cand_corpus(const CandCorpusParams &P, int row, int sm_count, cudaStream_t st) {
	if (row == 32) return launch_walk(k_cand_corpus<32>, P, sm_count, st);
	if (row == 16) return launch_walk(k_cand_corpus<16>, P, sm_count, st);
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
	__shared__ long long s_corp[CORP_EX];
	build_report(F, corp, s_corp);
}

cudaError_t run_cand_corpus_report(long long *blk, uint32_t C, apo_corpus_report *out, cudaStream_t st) {
	if (C == 0) return cudaSuccess;
	k_cand_corpus_report<<<C, 32, 0, st>>>(blk, blk + (uint64_t)C * CC_WORDS, out);
	return cudaGetLastError();
}

// ================================================================ per-candidate extremes (APO_SCORE_CANDIDATE_EXTREMES)
//   k_cand_extremes<Loader, TABLE, RECIP>  one pass over the evaluations a scoring call reads, on the shared loaders and
//                                          walk: every warp keeps the 32 smallest keys of each list of its current
//                                          candidate in registers (lane i holds the i-th) and writes them to its segment
//                                          slot when the candidate changes
//   k_cand_extremes_merge                  one warp per candidate: the persistent lists merged with the segments of the
//                                          warps whose tile range covers the candidate, in warp order
// No locks and no atomics: a warp's candidates form a range [c_lo(w), c_hi(w)] with c_lo(w + 1) >= c_hi(w), so the slots
// w + c of different warps never meet, and the merge finds the warps of a row by the pass's own range formula.
struct XKey { unsigned long long v, p; };
constexpr unsigned FULL = 0xffffffffu;
__device__ __forceinline__ bool xlt(const XKey &a, const XKey &b) { return a.v < b.v || (a.v == b.v && a.p < b.p); }
__device__ __forceinline__ XKey xshfl(const XKey &k, int src) { return {__shfl_sync(FULL, k.v, src), __shfl_sync(FULL, k.p, src)}; }
__device__ __forceinline__ XKey xshfl_xor(const XKey &k, int m) { return {__shfl_xor_sync(FULL, k.v, m), __shfl_xor_sync(FULL, k.p, m)}; }
__device__ __forceinline__ XKey xempty() { return {~0ull, ~0ull}; }

// order-preserving u64 of a binary64 value (-0.0 taken as +0.0)
__device__ __forceinline__ unsigned long long order_key(double x) {
	const unsigned long long u = (unsigned long long)__double_as_longlong(x == 0.0 ? 0.0 : x);
	return (u >> 63) ? ~u : (u | (1ull << 63));
}

// one key per lane -> ascending across the warp (bitonic sort, 15 compare-exchange steps)
__device__ __forceinline__ XKey warp_sort(XKey k, int lane) {
#pragma unroll
	for (int s = 2; s <= 32; s <<= 1) {
#pragma unroll
		for (int j = s >> 1; j > 0; j >>= 1) {
			const XKey o = xshfl_xor(k, j);
			const bool want_min = ((lane & j) == 0) == ((lane & s) == 0);
			if (want_min ? xlt(o, k) : xlt(k, o)) k = o;
		}
	}
	return k;
}

// list <- the 32 smallest of list and s, both ascending across the warp: the lane-wise min against s reversed is bitonic,
// five compare-exchange steps sort it
__device__ __forceinline__ XKey warp_merge(XKey list, const XKey &s, int lane) {
	const XKey r = xshfl(s, 31 - lane);
	XKey m = xlt(r, list) ? r : list;
#pragma unroll
	for (int j = 16; j > 0; j >>= 1) {
		const XKey o = xshfl_xor(m, j);
		if ((lane & j) ? xlt(m, o) : xlt(o, m)) m = o;
	}
	return m;
}

// offer one new key per lane to an ascending list: sort and merge only when some key beats the list's last entry
__device__ __forceinline__ void offer(XKey &list, const XKey &k, int lane) {
	const XKey last = xshfl(list, 31);
	if (__ballot_sync(FULL, xlt(k, last))) list = warp_merge(list, warp_sort(k, lane), lane);
}

__device__ __forceinline__ void store_lists(unsigned long long *slot, const XKey &lo, const XKey &hi, int lane) {
	reinterpret_cast<ulonglong2 *>(slot)[lane] = make_ulonglong2(lo.v, lo.p);
	reinterpret_cast<ulonglong2 *>(slot)[32 + lane] = make_ulonglong2(hi.v, hi.p);
}
__device__ __forceinline__ void load_lists(const unsigned long long *slot, XKey &lo, XKey &hi, int lane) {
	const ulonglong2 a = reinterpret_cast<const ulonglong2 *>(slot)[lane], b = reinterpret_cast<const ulonglong2 *>(slot)[32 + lane];
	lo = {a.x, a.y}; hi = {b.x, b.y};
}

template <class L, int TABLE, bool RECIP>
__global__ void __launch_bounds__(CB_THREADS, L::MIN_CTAS)
k_cand_extremes(const CandExtParams X, uint32_t tiles_per_cand, uint64_t total_tiles) {
	const CandEvals &P = X.src;
	__shared__ CandSmem S;
	__shared__ double s_rc[512];                                        // reciprocal of the total weight (div_lut)
	stage_tables<TABLE, true>(P, S, s_rc);
	const int lane = threadIdx.x & 31;
	XKey low = xempty(), high = xempty();

	auto flush = [&](uint32_t c) {
		store_lists(X.seg + (cand_warp() + c) * CX_WORDS, low, high, lane);
		low = high = xempty();
	};
	auto each = [&](uint32_t, uint64_t t, bool in, const typename L::Raw &R, uint32_t) {
		XKey kl = xempty(), kh = xempty();
		if (in) {
			CandEval E;
			L::decode(P, S, R, E);
			if (E.valid) {
				const unsigned long long k = order_key(cand_final_reward<RECIP>(E, X.W, S.tw, s_rc));
				kl = {k, P.idx_base + t};
				kh = {~k, P.idx_base + t};
			}
		}
		offer(low, kl, lane);
		offer(high, kh, lane);
	};
	cand_walk<L, 0>(P, tiles_per_cand, total_tiles, each, flush);
}

// the warp of the pass whose tile range holds `tile`: the largest w with total * w / nwarps <= tile
__device__ __forceinline__ uint64_t tile_owner(uint64_t tile, uint64_t total_tiles, uint64_t nwarps) {
	return ((tile + 1) * nwarps - 1) / total_tiles;
}

__global__ void __launch_bounds__(256)
k_cand_extremes_merge(unsigned long long *lists, const unsigned long long *seg, uint32_t C, uint32_t tiles_per_cand,
                      uint64_t total_tiles, uint64_t nwarps) {
	const uint32_t c = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
	if (c >= C) return;
	const int lane = threadIdx.x & 31;
	XKey low, high;
	load_lists(lists + (uint64_t)c * CX_WORDS, low, high, lane);
	const uint64_t w0 = tile_owner((uint64_t)c * tiles_per_cand, total_tiles, nwarps);
	const uint64_t w1 = tile_owner((uint64_t)(c + 1) * tiles_per_cand - 1, total_tiles, nwarps);
	for (uint64_t w = w0; w <= w1; w++) {
		if (total_tiles * w / nwarps == total_tiles * (w + 1) / nwarps) continue;   // a warp without tiles wrote no segment
		XKey sl, sh;
		load_lists(seg + (w + c) * CX_WORDS, sl, sh, lane);
		if (xlt(xshfl(sl, 0), xshfl(low, 31))) low = warp_merge(low, sl, lane);
		if (xlt(xshfl(sh, 0), xshfl(high, 31))) high = warp_merge(high, sh, lane);
	}
	store_lists(lists + (uint64_t)c * CX_WORDS, low, high, lane);
}

// the walk, then the merge of its segments into the persistent lists
template <class L, int TABLE, bool RECIP>
static cudaError_t launch_pass(const CandExtParams &X, int sm_count, cudaStream_t st) {
	Walk w;
	cudaError_t err = walk_grid(k_cand_extremes<L, TABLE, RECIP>, X.src, sm_count, w);
	if (err != cudaSuccess || w.grid == 0) return err;
	const uint64_t nwarps = w.grid * CB_WARPS;
	if (nwarps > CX_MAX_WARPS_PER_SM * (uint64_t)sm_count) return cudaErrorInvalidConfiguration;   // more than the segment slots hold
	k_cand_extremes<L, TABLE, RECIP><<<(unsigned)w.grid, CB_THREADS, 0, st>>>(X, w.tiles_per_cand, w.total_tiles);
	if ((err = cudaGetLastError()) != cudaSuccess) return err;
	k_cand_extremes_merge<<<(X.src.C + 7) / 8, 256, 0, st>>>(X.lists, X.seg, X.src.C, w.tiles_per_cand, w.total_tiles, nwarps);
	return cudaGetLastError();
}

// ================================================================ per-candidate group scores (APO_SCORE_CANDIDATE_GROUPS)
//   k_cand_groups<Loader, TABLE, RECIP>  one pass over the evaluations a scoring call reads, on the shared loaders and
//                                        walk: every group of 32 evaluations is split by the labels of its records
//   k_cand_groups_report                 words -> apo_group_score[C][G] with the breakdown's report rules
// A group of 32 evaluations is aggregated per label before it touches memory: the lanes that share a label (all 32 on the
// fast path, __match_any_sync otherwise) reduce their terms with __reduce_add_sync, and the lowest of them adds the sums into
// the warp's own shared accumulators of that label.  A term rint(fr * 2^52) enters as four 16-bit pieces of its two's
// complement and a sign count, so 32 of them sum exactly in 32 bits whatever the labels are; the warp's accumulators hold a
// run of CB_RUN_TILES tiles exactly (l0, l1 < 2^58, counts < 2^27) and are flushed into the (c, g) words when the candidate
// changes and at the breakdown's run limit.  A flush forms the run's signed sum l0 + 2^32 l1 - 2^64 neg (|sum| < 2^123) and
// adds it in the scoring partials' limb split (add_i128): words 0 and 1 grow by < 2^32 per flush, as the host bounds them.
struct GroupSmem {
	unsigned long long l0[CB_WARPS][APO_GROUPS_MAX], l1[CB_WARPS][APO_GROUPS_MAX];   // 2^0 and 2^32 limbs of the sum
	uint32_t n[CB_WARPS][APO_GROUPS_MAX], good[CB_WARPS][APO_GROUPS_MAX], bad[CB_WARPS][APO_GROUPS_MAX];
	uint32_t rew[CB_WARPS][APO_GROUPS_MAX], neg[CB_WARPS][APO_GROUPS_MAX];           // non-null terms, negative terms
};
// the fields of one evaluation (and, after __reduce_add_sync, of up to 32), 6 bits each
constexpr int GP_N = 0, GP_GOOD = 6, GP_BAD = 12, GP_REW = 18, GP_NEG = 24;

template <class L, int TABLE, bool RECIP>
__global__ void __launch_bounds__(CB_THREADS, L::MIN_CTAS)
k_cand_groups(const CandGroupParams X, uint32_t tiles_per_cand, uint64_t total_tiles) {
	const CandEvals &P = X.src;
	__shared__ CandSmem S;
	__shared__ double s_rc[512];                                        // reciprocal of the total weight (div_lut)
	__shared__ GroupSmem A;
	const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
	for (int g = lane; g < APO_GROUPS_MAX; g += 32) {
		A.l0[wp][g] = A.l1[wp][g] = 0ull;
		A.n[wp][g] = A.good[wp][g] = A.bad[wp][g] = A.rew[wp][g] = A.neg[wp][g] = 0u;
	}
	stage_tables<TABLE, true>(P, S, s_rc);
	const uint8_t *labels = X.labels + P.idx_base;
	const uint32_t G = X.G;

	auto flush = [&](uint32_t c) {
		__syncwarp();
		for (uint32_t g = lane; g < G; g += 32) {
			unsigned long long *w = (unsigned long long *)X.words + ((uint64_t)c * G + g) * GR_WORDS;
			const uint32_t neg = A.neg[wp][g], rew = A.rew[wp][g], n = A.n[wp][g], good = A.good[wp][g], bad = A.bad[wp][g];
			// each negative term carries -2^64
			add_i128((long long *)w, (__int128)A.l0[wp][g] + ((__int128)A.l1[wp][g] << 32) - ((__int128)neg << 64));
			if (rew) atomicAdd(w + 3, (unsigned long long)rew);
			if (n) atomicAdd(w + GR_TALLY, (unsigned long long)n);
			if (good) atomicAdd(w + GR_TALLY + 1, (unsigned long long)good);
			if (bad) atomicAdd(w + GR_TALLY + 2, (unsigned long long)bad);
			A.l0[wp][g] = A.l1[wp][g] = 0ull;
			A.n[wp][g] = A.good[wp][g] = A.bad[wp][g] = A.rew[wp][g] = A.neg[wp][g] = 0u;
		}
		__syncwarp();
	};
	// l: the label, fetched with the evaluation (past the row end: label 0, nothing added)
	auto each = [&](uint32_t, uint64_t, bool in, const typename L::Raw &R, uint32_t l) {
		uint32_t pk = 0;
		unsigned long long x = 0ull;
		if (in) {
			CandEval E;
			L::decode(P, S, R, E);
			pk = (1u << GP_N) | ((E.fb == 1u ? 1u : 0u) << GP_GOOD) | ((E.fb == 2u ? 1u : 0u) << GP_BAD);
			if (E.valid) {
				const long long fx = to_fx(cand_final_reward<RECIP>(E, X.W, S.tw, s_rc));
				x = (unsigned long long)fx;
				pk |= (1u << GP_REW) | ((fx < 0 ? 1u : 0u) << GP_NEG);
			}
		}
		const uint32_t peers = __all_sync(FULL, l == __shfl_sync(FULL, l, 0)) ? FULL : __match_any_sync(FULL, l);
		uint32_t s0 = (uint32_t)x & 0xFFFFu, s1 = (uint32_t)(x >> 16) & 0xFFFFu, s2 = (uint32_t)(x >> 32) & 0xFFFFu;
		uint32_t s3 = (uint32_t)(x >> 48), sp = pk;
		if (peers != (1u << lane)) {                                    // a label of its own needs no reduction: the
			s0 = __reduce_add_sync(peers, s0);                          // reductions run once per distinct peer mask
			s1 = __reduce_add_sync(peers, s1);
			s2 = __reduce_add_sync(peers, s2);
			s3 = __reduce_add_sync(peers, s3);
			sp = __reduce_add_sync(peers, sp);
		}
		if (lane == __ffs((int)peers) - 1) {                          // the lowest lane of the label: one writer per label
			A.l0[wp][l] += (unsigned long long)s0 + ((unsigned long long)s1 << 16);
			A.l1[wp][l] += (unsigned long long)s2 + ((unsigned long long)s3 << 16);
			A.n[wp][l] += (sp >> GP_N) & 63u;
			A.good[wp][l] += (sp >> GP_GOOD) & 63u;
			A.bad[wp][l] += (sp >> GP_BAD) & 63u;
			A.rew[wp][l] += (sp >> GP_REW) & 63u;
			A.neg[wp][l] += (sp >> GP_NEG) & 63u;
		}
		__syncwarp();                                                   // the next group's writer of a label may be another lane
	};
	cand_walk<L, CB_RUN_TILES>(P, tiles_per_cand, total_tiles, each, flush, [&](uint64_t t) { return (uint32_t)__ldg(labels + t); });
}

// one thread per (c, g)
__global__ void __launch_bounds__(256)
k_cand_groups_report(const long long *words, uint64_t n, apo_group_score *out) {
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const long long *w = words + i * GR_WORDS;
	apo_group_score R;
	R.total = (uint64_t)w[GR_TALLY];
	R.good = (uint64_t)w[GR_TALLY + 1];
	R.bad = (uint64_t)w[GR_TALLY + 2];
	R.goodRate = report_good_rate(R.good, R.bad);
	R.withReward = (uint64_t)w[3];
	R.rewardSum = limbs_to_double(w);                                   // the scoring partials' limbs, as k_cand_report reads them
	R.avgReward = report_avg_reward(R.rewardSum, R.withReward);
	out[i] = R;
}

cudaError_t run_cand_groups_report(const long long *words, uint32_t C, uint32_t G, apo_group_score *out, cudaStream_t st) {
	const uint64_t n = (uint64_t)C * G;
	if (n == 0) return cudaSuccess;
	k_cand_groups_report<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(words, n, out);
	return cudaGetLastError();
}

// ================================================================ per-candidate reward spread (APO_SCORE_CANDIDATE_SPREAD)
//   k_cand_spread<Loader, TABLE, RECIP>  one pass over the evaluations a scoring call reads, on the shared loaders and walk:
//                                        every lane sums x^2 exactly, x = rint(fr * 2^52) the term the call summed
//   k_cand_spread_report                 n and S1 from the scoring call's partials, S2 from the words -> apo_candidate_spread
// |x| <= 2^61 in the scoring domain (a term outside it fails the call), so x^2 < 2^127 is one exact unsigned 128-bit product
// and a lane's 192-bit sum holds a run of CB_RUN_TILES tiles (2^21 terms) with room to spare.  A flush reduces the warp's sums
// and adds the result into the candidate's three words with carried atomics: exact modulo 2^192 for any number of flushes,
// and S2 < 2^192 for any n < 2^64.
struct U192 { unsigned long long w0, w1, w2; };

__device__ __forceinline__ void u192_add(U192 &a, unsigned long long w0, unsigned long long w1, unsigned long long w2) {
	asm("add.cc.u64 %0, %0, %3;\n\taddc.cc.u64 %1, %1, %4;\n\taddc.u64 %2, %2, %5;" : "+l"(a.w0), "+l"(a.w1), "+l"(a.w2) : "l"(w0), "l"(w1), "l"(w2));
}

// a += x^2
__device__ __forceinline__ void u192_add_sq(U192 &a, long long x) {
	const unsigned long long u = x < 0 ? 0ull - (unsigned long long)x : (unsigned long long)x;
	unsigned long long lo, hi;
	asm("mul.lo.u64 %0, %2, %2;\n\tmul.hi.u64 %1, %2, %2;" : "=l"(lo), "=l"(hi) : "l"(u));
	u192_add(a, lo, hi, 0ull);
}

// w[0..2] += v modulo 2^192: every atomic returns the word it added to, so its carry out is known exactly
__device__ __forceinline__ void atomic_add_u192(unsigned long long *w, const U192 &v) {
	unsigned long long c1 = 0ull, c2 = 0ull;
	if (v.w0) { const unsigned long long o = atomicAdd(w, v.w0); c1 = o + v.w0 < o ? 1ull : 0ull; }
	const unsigned long long m = v.w1 + c1;
	c2 = m < c1 ? 1ull : 0ull;                                          // v.w1 all ones plus the carry
	if (m) { const unsigned long long o = atomicAdd(w + 1, m); c2 += o + m < o ? 1ull : 0ull; }
	const unsigned long long h = v.w2 + c2;
	if (h) atomicAdd(w + 2, h);
}

template <class L, int TABLE, bool RECIP>
__global__ void __launch_bounds__(CB_THREADS, L::MIN_CTAS)
k_cand_spread(const CandSpreadParams X, uint32_t tiles_per_cand, uint64_t total_tiles) {
	const CandEvals &P = X.src;
	__shared__ CandSmem S;
	__shared__ double s_rc[512];                                        // reciprocal of the total weight (div_lut)
	stage_tables<TABLE, true>(P, S, s_rc);
	const int lane = threadIdx.x & 31;
	U192 a{0ull, 0ull, 0ull};

	auto flush = [&](uint32_t c) {
		U192 s = a;
#pragma unroll
		for (int o = 16; o > 0; o >>= 1)                                // 32 lanes of < 2^148 each: no carry leaves the sum
			u192_add(s, __shfl_xor_sync(FULL, s.w0, o), __shfl_xor_sync(FULL, s.w1, o), __shfl_xor_sync(FULL, s.w2, o));
		if (lane == 0 && (s.w0 | s.w1 | s.w2)) atomic_add_u192(X.words + (uint64_t)c * SP_WORDS, s);
		a = U192{0ull, 0ull, 0ull};
	};
	auto each = [&](uint32_t, uint64_t, bool in, const typename L::Raw &R, uint32_t) {
		if (!in) return;
		CandEval E;
		L::decode(P, S, R, E);
		if (E.valid) u192_add_sq(a, to_fx(cand_final_reward<RECIP>(E, X.W, S.tw, s_rc)));
	};
	cand_walk<L, CB_RUN_TILES>(P, tiles_per_cand, total_tiles, each, flush);
}

// ---- exact 256-bit arithmetic of the report (little-endian words)
// m += v * 2^(64 k)
__device__ __forceinline__ void u256_add_at(unsigned long long m[4], unsigned __int128 v, int k) {
	unsigned __int128 carry = v;
	for (int i = k; i < 4 && carry; i++) {
		const unsigned __int128 s = (unsigned __int128)m[i] + (unsigned long long)carry;
		m[i] = (unsigned long long)s;
		carry = (carry >> 64) + (s >> 64);
	}
}

// RN(m) as binary64: the 64 bits below the leading one, the discarded bits ORed into the last of them (a sticky bit well below
// the rounding position), then one correctly rounded conversion and an exact scaling
__device__ __forceinline__ double u256_to_double(const unsigned long long m[4]) {
	int k = 3;
	while (k > 0 && m[k] == 0ull) k--;
	if (k == 0) return __ull2double_rn(m[0]);
	const int sh = 64 * k - __clzll((long long)m[k]);                 // bit index of the lowest of the 64 kept bits, >= 1
	const int q = sh >> 6, b = sh & 63;
	unsigned long long top = b ? (m[q] >> b) | (m[q + 1] << (64 - b)) : m[q];
	bool sticky = b ? (m[q] << (64 - b)) != 0ull : false;
	for (int i = 0; i < q; i++) sticky |= m[i] != 0ull;
	return ldexp(__ull2double_rn(top | (sticky ? 1ull : 0ull)), sh);
}

// variance, stdDev and stdErr of n terms with the exact sums s1 (|s1| < 2^128) and s2 (< 2^192): M = n * s2 - s1^2 in 256
// bits, rounded once (the spread's rules, and the paired comparison's with d for x)
__device__ __forceinline__ void spread_moments(uint64_t n, __int128 s1, const unsigned long long s2[4], double &variance, double &stdDev,
                                               double &stdErr) {
	if (n < 2) {
		variance = stdDev = stdErr = __longlong_as_double(0x7ff8000000000000ll);
		return;
	}
	// M = n * S2 - S1^2, with n * S2 < 2^256 and |S1| < 2^128
	unsigned long long a[4] = {0ull, 0ull, 0ull, 0ull}, b[4] = {0ull, 0ull, 0ull, 0ull};
	for (int i = 0; i < 3; i++) u256_add_at(a, (unsigned __int128)n * s2[i], i);
	const unsigned __int128 u = s1 < 0 ? (unsigned __int128)0 - (unsigned __int128)s1 : (unsigned __int128)s1;
	const unsigned long long u0 = (unsigned long long)u, u1 = (unsigned long long)(u >> 64);
	u256_add_at(b, (unsigned __int128)u0 * u0, 0);
	u256_add_at(b, (unsigned __int128)u0 * u1, 1);
	u256_add_at(b, (unsigned __int128)u0 * u1, 1);
	u256_add_at(b, (unsigned __int128)u1 * u1, 2);
	unsigned long long m[4], borrow = 0ull;
	for (int i = 0; i < 4; i++) {
		const unsigned long long d = a[i] - b[i];
		const unsigned long long nb = (a[i] < b[i] ? 1ull : 0ull) | (d < borrow ? 1ull : 0ull);
		m[i] = d - borrow;
		borrow = nb;
	}
	const double dn = __ull2double_rn(n);
	variance = __ddiv_rn(__ddiv_rn(__dmul_rn(u256_to_double(m), 0x1p-104), dn), __ull2double_rn(n - 1));
	stdDev = __dsqrt_rn(variance);
	stdErr = __dsqrt_rn(__ddiv_rn(variance, dn));
}

// one thread per candidate
__global__ void __launch_bounds__(256)
k_cand_spread_report(const unsigned long long *words, const long long *partials, uint32_t C, struct apo_candidate_spread *out) {
	const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
	if (c >= C) return;
	long long l[4];
#pragma unroll
	for (int q = 0; q < 4; q++) l[q] = partials[(uint64_t)ACC_PER_CAND * c + q];
	const uint64_t n = (uint64_t)l[3];
	const __int128 s1 = ((__int128)l[2] << 64) + ((__int128)l[1] << 32) + (__int128)l[0];
	const unsigned long long *w = words + (uint64_t)c * SP_WORDS;
	const unsigned long long s2[4] = {w[0], w[1], w[2], 0ull};
	struct apo_candidate_spread R;
	R.n = n;
	R.sumLo = (uint64_t)(unsigned __int128)s1;
	R.sumHi = (int64_t)(s1 >> 64);
	R.sumSq[0] = s2[0]; R.sumSq[1] = s2[1]; R.sumSq[2] = s2[2];
	R.mean = report_avg_reward(limbs_to_double(l), n);                   // the division scores[c] is: same bits
	R.rewardSumSq = __dmul_rn(u256_to_double(s2), 0x1p-104);
	spread_moments(n, s1, s2, R.variance, R.stdDev, R.stdErr);
	out[c] = R;
}

cudaError_t run_cand_spread_report(const unsigned long long *words, const long long *partials, uint32_t C, struct apo_candidate_spread *out,
                                   cudaStream_t st) {
	if (C == 0) return cudaSuccess;
	k_cand_spread_report<<<(C + 255) / 256, 256, 0, st>>>(words, partials, C, out);
	return cudaGetLastError();
}

// ================================================================ paired comparison with a reference (APO_SCORE_CANDIDATE_PAIRS)
//   k_cand_pairs<Loader, TABLE, RECIP>  one pass over the evaluations a scoring call reads, on the shared loaders and walk:
//                                       the walk fetches the reference's row with the candidate's own, and every lane compares
//                                       the two terms x = rint(fr * 2^52) the call summed at each position
//   k_cand_pair_report                  the pass's words -> apo_candidate_pair
// Per lane and run of at most CB_RUN_TILES tiles (2^21 positions): the five tallies as u32, D1 as a signed 128-bit sum
// (|d| <= 2^62, so |run| < 2^83) and D2 as an unsigned 192-bit one (d^2 <= 2^124).  A flush reduces the warp's sums, D1
// sign-extended to 192 bits, and adds them into the candidate's words with carried atomics, exact modulo 2^192 for any
// number of flushes (|D1| < 2^126 and D2 < 2^192 for any n < 2^64), and the tallies as u64 atomics.  No word takes 32-bit
// limbs that a reader would need carried, so the host's limb carry (limb_guard) has nothing of this pass to rewrite.

// the row of c's reference in this launch (the host keeps every reference inside the launch's candidates).  Two rows in flight
// per group: loaders of more than 16 bytes per evaluation (Form D's 36, Form R's 32) keep 2 groups, so that the lane holds the
// bytes one row holds at their U (Form D at U = 4 and two rows reaches the 128-register bound of two CTAs per SM and spills)
struct RefRow {
	static constexpr bool PAIR = true;
	template <class L> static constexpr int U = sizeof(typename L::Raw) > 16 ? 2 : L::U;
	const uint32_t *refs;
	uint32_t base;
	__device__ uint32_t operator()(uint32_t c) const {
		const uint32_t r = __ldg(refs + c);
		return r == APO_PAIR_NONE ? APO_PAIR_NONE : r - base;
	}
};

template <class L, int TABLE, bool RECIP>
__global__ void __launch_bounds__(CB_THREADS, L::MIN_CTAS)
k_cand_pairs(const CandPairParams X, uint32_t tiles_per_cand, uint64_t total_tiles) {
	const CandEvals &P = X.src;
	__shared__ CandSmem S;
	__shared__ double s_rc[512];                                        // reciprocal of the total weight (div_lut)
	stage_tables<TABLE, true>(P, S, s_rc);
	const int lane = threadIdx.x & 31;
	Acc128 d1;
	d1.zero();
	U192 d2{0ull, 0ull, 0ull};
	uint32_t wins = 0, losses = 0, ties = 0, conly = 0, ronly = 0;

	auto flush = [&](uint32_t c) {
		U192 s1{d1.lo, (unsigned long long)d1.hi, (unsigned long long)(d1.hi >> 63)}, s2 = d2;
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) {                              // exact: 32 lanes of |D1| < 2^83 and D2 < 2^145
			u192_add(s1, __shfl_xor_sync(FULL, s1.w0, o), __shfl_xor_sync(FULL, s1.w1, o), __shfl_xor_sync(FULL, s1.w2, o));
			u192_add(s2, __shfl_xor_sync(FULL, s2.w0, o), __shfl_xor_sync(FULL, s2.w1, o), __shfl_xor_sync(FULL, s2.w2, o));
		}
		const uint32_t k[5] = {warp_sum_u32(wins), warp_sum_u32(losses), warp_sum_u32(ties), warp_sum_u32(conly), warp_sum_u32(ronly)};
		if (lane == 0) {
			unsigned long long *w = X.words + (uint64_t)c * PR_WORDS;
			if (s1.w0 | s1.w1 | s1.w2) atomic_add_u192(w + PR_D1, s1);
			if (s2.w0 | s2.w1 | s2.w2) atomic_add_u192(w + PR_D2, s2);
#pragma unroll
			for (int i = 0; i < 5; i++)
				if (k[i]) atomicAdd(w + PR_CNT + i, (unsigned long long)k[i]);
		}
		d1.zero();
		d2 = U192{0ull, 0ull, 0ull};
		wins = losses = ties = conly = ronly = 0;
	};
	auto each = [&](uint32_t, uint64_t, bool in, const typename L::Raw &R, const typename L::Raw &Q, uint32_t) {
		if (!in) return;
		CandEval E;
		L::decode(P, S, R, E);
		const bool vc = E.valid != 0u;
		const long long xc = vc ? to_fx(cand_final_reward<RECIP>(E, X.W, S.tw, s_rc)) : 0ll;
		L::decode(P, S, Q, E);
		const bool vr = E.valid != 0u;
		const long long xr = vr ? to_fx(cand_final_reward<RECIP>(E, X.W, S.tw, s_rc)) : 0ll;
		if (vc && vr) {
			const long long d = xc - xr;
			wins += d > 0 ? 1u : 0u;
			losses += d < 0 ? 1u : 0u;
			ties += d == 0 ? 1u : 0u;
			d1.add(d);
			u192_add_sq(d2, d);
		} else {
			conly += vc ? 1u : 0u;
			ronly += vr ? 1u : 0u;
		}
	};
	cand_walk<L, CB_RUN_TILES>(P, tiles_per_cand, total_tiles, each, flush, NoSide{}, RefRow{X.refs, X.base});
}

// one comparison's words (PR_WORDS) and reference -> apo_candidate_pair, for the whole record axis or one group of it
__device__ __forceinline__ void pair_report(const unsigned long long *w, uint32_t ref, struct apo_candidate_pair *out) {
	struct apo_candidate_pair R;
	R.ref = ref;
	R.pad = 0u;
	R.wins = w[PR_CNT]; R.losses = w[PR_CNT + 1]; R.ties = w[PR_CNT + 2]; R.candOnly = w[PR_CNT + 3]; R.refOnly = w[PR_CNT + 4];
	const uint64_t n = R.wins + R.losses + R.ties;
	R.n = n;
	const __int128 s1 = (__int128)(((unsigned __int128)w[PR_D1 + 1] << 64) | w[PR_D1]);   // word 2 is the sign extension
	R.sumLo = w[PR_D1];
	R.sumHi = (int64_t)w[PR_D1 + 1];
	const unsigned long long s2[4] = {w[PR_D2], w[PR_D2 + 1], w[PR_D2 + 2], 0ull};
	R.sumSq[0] = s2[0]; R.sumSq[1] = s2[1]; R.sumSq[2] = s2[2];
	const long long l[4] = {(long long)(s1 & 0xFFFFFFFF), (long long)((s1 >> 32) & 0xFFFFFFFF), (long long)(s1 >> 64), 0ll};
	R.meanDiff = report_avg_reward(limbs_to_double(l), n);               // the rounding sequence of scores[c]
	spread_moments(n, s1, s2, R.variance, R.stdDev, R.stdErr);
	*out = R;
}

// one thread per candidate
__global__ void __launch_bounds__(256)
k_cand_pair_report(const unsigned long long *words, const uint32_t *refs, uint32_t C, struct apo_candidate_pair *out) {
	const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
	if (c >= C) return;
	pair_report(words + (uint64_t)c * PR_WORDS, refs[c], out + c);
}

cudaError_t run_cand_pair_report(const unsigned long long *words, const uint32_t *refs, uint32_t C, struct apo_candidate_pair *out,
                                 cudaStream_t st) {
	if (C == 0) return cudaSuccess;
	k_cand_pair_report<<<(C + 255) / 256, 256, 0, st>>>(words, refs, C, out);
	return cudaGetLastError();
}

// ================================================================ paired comparison per record group (APO_SCORE_CANDIDATE_GROUP_PAIRS)
//   k_cand_group_pairs<Loader, TABLE, RECIP>  the paired comparison's pass split as the group scores split: the walk fetches
//                                             the reference's row and the position's label with the candidate's own row
//   k_cand_group_pairs_report                 words -> apo_candidate_pair[C][G] by the pair report's code (pair_report)
// A group of 32 positions is aggregated per label before it touches memory, as in k_cand_groups: the lanes that share a
// label (all 32 on the fast path, __match_any_sync otherwise; a lane alone in its label skips the reductions) reduce d as four
// 16-bit pieces of its two's complement, d^2 (< 2^124) as eight 16-bit pieces, every piece summing to < 2^21, and the five
// tallies in 6-bit fields of one word.  The lowest lane of the label adds them into the warp's accumulators of that label: D1
// as limbs of weight 2^0 and 2^32, each negative d carrying -2^64 (the negative d are the losses, so the losses count them),
// D2 as four limbs of weight 2^0, 2^32, 2^64 and 2^96.  Every limb grows by < 2^38 per group of 32, so by < 2^59 over a run of
// CB_RUN_TILES tiles (2^21 groups) whatever the labels.  A flush (candidate change, run limit, end of the range) forms every
// label's run D1 (signed) and D2 as 192-bit integers and adds them into the (c, g) words with the pairs' carried atomics: exact
// modulo 2^192 for any number of flushes.  No word takes 32-bit limbs, so limb_guard has nothing of this pass to rewrite.
// The accumulators are dynamic shared memory sized by G (gp_bytes): at G = 64 they and the staged tables pass the 48 KB a
// kernel may hold without opting in.
constexpr int GP_LIMBS = 6;                          // u64 per label and warp: D1 at 2^0, 2^32; D2 at 2^0, 2^32, 2^64, 2^96
constexpr int GP_TALLIES = 5;                        // u32 per label and warp: wins, losses, ties, candOnly, refOnly (PR_CNT order)
constexpr size_t gp_bytes(uint32_t G) { return (size_t)CB_WARPS * G * (GP_LIMBS * 8 + GP_TALLIES * 4); }

template <class L, int TABLE, bool RECIP>
__global__ void __launch_bounds__(CB_THREADS, L::MIN_CTAS)
k_cand_group_pairs(const CandGroupPairParams X, uint32_t tiles_per_cand, uint64_t total_tiles) {
	const CandEvals &P = X.src;
	__shared__ CandSmem S;
	__shared__ double s_rc[512];                                        // reciprocal of the total weight (div_lut)
	extern __shared__ unsigned long long gp_acc[];                      // [GP_LIMBS][CB_WARPS][G] u64, then [GP_TALLIES][CB_WARPS][G] u32
	const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
	const uint32_t G = X.G, WG = CB_WARPS * G;
	unsigned long long *limb = gp_acc + wp * G;                         // limb k of label l: limb[k * WG + l]
	uint32_t *tally = reinterpret_cast<uint32_t *>(gp_acc + GP_LIMBS * WG) + wp * G;
	for (uint32_t g = lane; g < G; g += 32) {
		for (int k = 0; k < GP_LIMBS; k++) limb[k * WG + g] = 0ull;
		for (int k = 0; k < GP_TALLIES; k++) tally[k * WG + g] = 0u;
	}
	stage_tables<TABLE, true>(P, S, s_rc);
	const uint8_t *labels = X.labels + P.idx_base;

	auto flush = [&](uint32_t c) {
		__syncwarp();
		for (uint32_t g = lane; g < G; g += 32) {
			unsigned long long *w = X.words + ((uint64_t)c * G + g) * PR_WORDS;
			const __int128 d1 = (__int128)limb[g] + ((__int128)limb[WG + g] << 32) - ((__int128)tally[WG + g] << 64);   // |d1| < 2^92
			const U192 s1{(unsigned long long)d1, (unsigned long long)(d1 >> 64), (unsigned long long)(d1 >> 127)};
			const unsigned __int128 lo = (unsigned __int128)limb[2 * WG + g] + ((unsigned __int128)limb[3 * WG + g] << 32);
			const unsigned __int128 hi = (unsigned __int128)limb[4 * WG + g] + ((unsigned __int128)limb[5 * WG + g] << 32) + (lo >> 64);
			const U192 s2{(unsigned long long)lo, (unsigned long long)hi, (unsigned long long)(hi >> 64)};
			if (s1.w0 | s1.w1 | s1.w2) atomic_add_u192(w + PR_D1, s1);
			if (s2.w0 | s2.w1 | s2.w2) atomic_add_u192(w + PR_D2, s2);
			for (int k = 0; k < GP_TALLIES; k++) {
				if (const uint32_t v = tally[k * WG + g]) atomicAdd(w + PR_CNT + k, (unsigned long long)v);
				tally[k * WG + g] = 0u;
			}
			for (int k = 0; k < GP_LIMBS; k++) limb[k * WG + g] = 0ull;
		}
		__syncwarp();
	};
	// l: the label, fetched with the evaluations (past the row end: label 0, nothing added)
	auto each = [&](uint32_t, uint64_t, bool in, const typename L::Raw &R, const typename L::Raw &Q, uint32_t l) {
		unsigned long long u = 0ull, q0 = 0ull, q1 = 0ull;              // d as two's complement, d^2 as two words
		uint32_t pk = 0u;                                                // the tallies, 6 bits each in PR_CNT order
		if (in) {
			CandEval E;
			L::decode(P, S, R, E);
			const bool vc = E.valid != 0u;
			const long long xc = vc ? to_fx(cand_final_reward<RECIP>(E, X.W, S.tw, s_rc)) : 0ll;
			L::decode(P, S, Q, E);
			const bool vr = E.valid != 0u;
			const long long xr = vr ? to_fx(cand_final_reward<RECIP>(E, X.W, S.tw, s_rc)) : 0ll;
			if (vc && vr) {
				const long long d = xc - xr;
				pk = 1u << (d > 0 ? 0 : d < 0 ? 6 : 12);
				u = (unsigned long long)d;
				const unsigned long long a = d < 0 ? 0ull - u : u;
				asm("mul.lo.u64 %0, %2, %2;\n\tmul.hi.u64 %1, %2, %2;" : "=l"(q0), "=l"(q1) : "l"(a));
			} else {
				pk = ((vc ? 1u : 0u) << 18) | ((vr ? 1u : 0u) << 24);
			}
		}
		const uint32_t peers = __all_sync(FULL, l == __shfl_sync(FULL, l, 0)) ? FULL : __match_any_sync(FULL, l);
		uint32_t p[13];                                                  // d: p[0..3], d^2: p[4..11], tallies: p[12]
#pragma unroll
		for (int k = 0; k < 4; k++) {
			p[k] = (uint32_t)(u >> (16 * k)) & 0xFFFFu;
			p[4 + k] = (uint32_t)(q0 >> (16 * k)) & 0xFFFFu;
			p[8 + k] = (uint32_t)(q1 >> (16 * k)) & 0xFFFFu;
		}
		p[12] = pk;
		if (peers != (1u << lane)) {                                    // a label of its own needs no reduction
#pragma unroll
			for (int k = 0; k < 13; k++) p[k] = __reduce_add_sync(peers, p[k]);
		}
		if (lane == __ffs((int)peers) - 1) {                          // the lowest lane of the label: one writer per label
#pragma unroll
			for (int k = 0; k < GP_LIMBS; k++) limb[k * WG + l] += (unsigned long long)p[2 * k] + ((unsigned long long)p[2 * k + 1] << 16);
#pragma unroll
			for (int k = 0; k < GP_TALLIES; k++) tally[k * WG + l] += (p[12] >> (6 * k)) & 63u;
		}
		__syncwarp();                                                   // the next group's writer of a label may be another lane
	};
	cand_walk<L, CB_RUN_TILES>(P, tiles_per_cand, total_tiles, each, flush, [&](uint64_t t) { return (uint32_t)__ldg(labels + t); },
	                           RefRow{X.refs, X.base});
}

// one thread per (c, g)
__global__ void __launch_bounds__(256)
k_cand_group_pairs_report(const unsigned long long *words, const uint32_t *refs, uint32_t G, uint64_t n, struct apo_candidate_pair *out) {
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	pair_report(words + i * PR_WORDS, refs[i / G], out + i);
}

cudaError_t run_cand_group_pairs_report(const unsigned long long *words, const uint32_t *refs, uint32_t C, uint32_t G,
                                        struct apo_candidate_pair *out, cudaStream_t st) {
	const uint64_t n = (uint64_t)C * G;
	if (n == 0) return cudaSuccess;
	k_cand_group_pairs_report<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(words, refs, G, n, out);
	return cudaGetLastError();
}

// ================================================================ limb carry of the words that accumulate across launches
// Every flush adds < 2^37 to the unsigned limbs l0 and l1 of a triple (flush_acc128: 32 lanes of < 2^32; add_i128: < 2^32),
// which every reader takes as signed int64.  One launch adds at most limb_flush_bound flushes into any one candidate's triple:
// one per warp (the scoring kernels run <= sm_count CTAs of <= 32 warps, the walks <= 64 resident warps per SM) plus the run
// limit's (the shortest, k_cand_corpus's CC_RUN_TILES, in tiles of CB_TILE evaluations).  The host sums the bound over the
// launches of a session or host-streaming call and, before it could pass LIMB_FLUSH_MAX, rewrites every triple to its value
// with l0, l1 < 2^32 (k_carry_limbs): then l0, l1 < 2^32 + LIMB_FLUSH_MAX * 2^37 < 2^63 at every read.
uint64_t limb_flush_bound(uint64_t count, int sm_count) {
	const uint64_t tiles = (count + CB_TILE - 1) / CB_TILE;
	return 64ull * (uint64_t)sm_count + tiles / CC_RUN_TILES + 1;
}

// one thread per triple: w + r * row_words + first + 4 k for r < rows, k < per_row
__global__ void __launch_bounds__(256)
k_carry_limbs(long long *w, uint64_t n, uint32_t row_words, uint32_t first, uint32_t per_row) {
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	long long *l = w + (i / per_row) * row_words + first + 4 * (i % per_row);
	const __int128 v = ((__int128)l[2] << 64) + ((__int128)l[1] << 32) + (__int128)l[0];
	l[0] = (long long)(v & 0xFFFFFFFF);
	l[1] = (long long)((v >> 32) & 0xFFFFFFFF);
	l[2] = (long long)(v >> 64);
}

cudaError_t run_carry_limbs(long long *w, uint64_t rows, uint32_t row_words, uint32_t first, uint32_t per_row, cudaStream_t st) {
	const uint64_t n = rows * per_row;
	if (n == 0) return cudaSuccess;
	k_carry_limbs<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(w, n, row_words, first, per_row);
	return cudaGetLastError();
}

// ================================================================ one dispatch for the passes that read every source
template <class L, int TABLE, bool>
static cudaError_t launch_pass(const CandParams &P, int sm_count, cudaStream_t st) {
	return launch_walk(k_cand_breakdown<L, TABLE>, P, sm_count, st);
}
template <class L, int TABLE, bool RECIP>
static cudaError_t launch_pass(const CandGroupParams &X, int sm_count, cudaStream_t st) {
	return launch_walk(k_cand_groups<L, TABLE, RECIP>, X, sm_count, st);
}
template <class L, int TABLE, bool RECIP>
static cudaError_t launch_pass(const CandSpreadParams &X, int sm_count, cudaStream_t st) {
	return launch_walk(k_cand_spread<L, TABLE, RECIP>, X, sm_count, st);
}
template <class L, int TABLE, bool RECIP>
static cudaError_t launch_pass(const CandPairParams &X, int sm_count, cudaStream_t st) {
	return launch_walk(k_cand_pairs<L, TABLE, RECIP>, X, sm_count, st);
}
template <class L, int TABLE, bool RECIP>
static cudaError_t launch_pass(const CandGroupPairParams &X, int sm_count, cudaStream_t st) {
	// the opt-in past 48 KB belongs to the current device's context: set once per device (ordinals past 63 set it every launch)
	static std::atomic<uint64_t> opted{0ull};
	int dev = 0;
	cudaError_t err = cudaGetDevice(&dev);
	if (err != cudaSuccess) return err;
	const uint64_t bit = dev >= 0 && dev < 64 ? 1ull << dev : 0ull;
	if (!bit || !(opted.load() & bit)) {
		err = cudaFuncSetAttribute(k_cand_group_pairs<L, TABLE, RECIP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gp_bytes(APO_GROUPS_MAX));
		if (err != cudaSuccess) return err;
		opted.fetch_or(bit);
	}
	return launch_walk(k_cand_group_pairs<L, TABLE, RECIP>, X, sm_count, st, gp_bytes(X.G));
}

// the loader of each source and the table it stages; RECIP: the division of the passes that divide (div_lut)
template <bool RECIP, class X>
static cudaError_t by_source(const X &x, int source, int sm_count, cudaStream_t st) {
	switch (source) {
	case CAND_DIMS: return launch_pass<LoadDims, 0, RECIP>(x, sm_count, st);
	case CAND_REC32: return launch_pass<LoadRec<32>, 0, RECIP>(x, sm_count, st);
	case CAND_REC16: return launch_pass<LoadRec<16>, 0, RECIP>(x, sm_count, st);
	case CAND_Q: return launch_pass<LoadQ, 1, RECIP>(x, sm_count, st);
	case CAND_T: return launch_pass<LoadT, 2, RECIP>(x, sm_count, st);
	case CAND_W: return launch_pass<LoadW, 1, RECIP>(x, sm_count, st);
	default: return cudaErrorInvalidValue;
	}
}

cudaError_t run_cand_breakdown(const CandParams &P, int source, int sm_count, cudaStream_t st) {
	return by_source<false>(P, source, sm_count, st);                  // the breakdown sums the dimensions: no division
}
cudaError_t run_cand_extremes(const CandExtParams &X, int source, bool recip, int sm_count, cudaStream_t st) {
	return recip ? by_source<true>(X, source, sm_count, st) : by_source<false>(X, source, sm_count, st);
}
cudaError_t run_cand_groups(const CandGroupParams &X, int source, bool recip, int sm_count, cudaStream_t st) {
	return recip ? by_source<true>(X, source, sm_count, st) : by_source<false>(X, source, sm_count, st);
}
cudaError_t run_cand_spread(const CandSpreadParams &X, int source, bool recip, int sm_count, cudaStream_t st) {
	return recip ? by_source<true>(X, source, sm_count, st) : by_source<false>(X, source, sm_count, st);
}
cudaError_t run_cand_pairs(const CandPairParams &X, int source, bool recip, int sm_count, cudaStream_t st) {
	return recip ? by_source<true>(X, source, sm_count, st) : by_source<false>(X, source, sm_count, st);
}
cudaError_t run_cand_group_pairs(const CandGroupPairParams &X, int source, bool recip, int sm_count, cudaStream_t st) {
	return recip ? by_source<true>(X, source, sm_count, st) : by_source<false>(X, source, sm_count, st);
}

}  // namespace apo
