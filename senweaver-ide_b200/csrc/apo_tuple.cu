// apo_tuple.cu — Form T: evaluations as indices into a dictionary of distinct evaluations, and K1t.
//
// The nine reward dimensions of one evaluation are functions of a handful of small counters (TCS:668-763): eight take
// <= 15 values, tool_success_rate a few hundred ratios.  Over C x T evaluations only 10^5 .. 10^6 DISTINCT evaluations
// occur (measured on the build's generator: 139 k in 48 M), and the frequent ones dominate (the 24 k most frequent cover
// 98.5 %).  Form T therefore keeps, per tensor,
//     tbook : the distinct evaluations as Form P pairs (code word + tool_success_rate index), most frequent first
// and per evaluation
//     tl/th : the 24-bit index of its entry as a 16-bit and an 8-bit plane                                   3 B
// instead of 36 B (Form D) / 14 B (Form Q) / 6 B (Form P).  finalReward of an entry is computed ONCE per scoring call by
// k_tuple_values with exactly the operations of K1q (product-table lookups in push order, the same division, the same
// rint(x * 2^52)), so summing table entries gives the integers K1 / K1q / the oracle produce: bit-exact by construction.
// K1t then is a gather-and-add: the hot head of the table in shared memory, the tail through L1/L2.
#include <cstdlib>
#include "apo_device.cuh"
#include "apo_corpus.cuh"
#include "apo_kernels.h"

namespace apo {

// =================================================================== dictionary entries -> table values
template <bool RECIP>
__global__ void __launch_bounds__(256)
k_tuple_values(const TupleValParams P) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i > P.n) return;
	if (i == P.n) { P.tval[i] = 0; return; }                      // sentinel: contributes nothing, counts nothing
	const uint32_t w = P.tb_pc[i];
	const uint32_t k2 = P.tb_pd[i] & 4095u;
	uint32_t code[8], mask = 0;
#pragma unroll
	for (int j = 0; j < 8; j++) {
		const uint32_t nib = (w >> (4 * j)) & 15u;
		code[j] = nib == 15u ? 255u : nib;                          // product table slot 255 holds +0.0, empty slots NaN
		mask |= (nib != 15u ? 1u : 0u) << (j < 2 ? j : j + 1);
	}
	const bool p2 = k2 != 4095u;
	mask |= (p2 ? 1u : 0u) << 2;
	const float d2f = p2 ? P.d2book[k2] : 0.0f;
	// TCS:777-783 in push order, the operations of evalq_ws (csrc/apo_compact.cu)
	double ws = P.ptab[0 * 256 + code[0]];
	ws = __dadd_rn(ws, P.ptab[1 * 256 + code[1]]);
	ws = __dadd_rn(ws, __dmul_rn((double)d2f, P.w2));
#pragma unroll
	for (int j = 2; j < 8; j++) ws = __dadd_rn(ws, P.ptab[j * 256 + code[j]]);
	const double2 t = make_double2(P.lut[mask], P.lut[512 + mask]);
	const double v = div_lut<RECIP>(ws, t);
	const long long fx = to_fx(v);
	const bool counted = t.x > 0.0;
	// ws is NaN when the entry names an empty or NaN slot of either codebook (the product table holds NaN there).
	// K1t adds up to 16 entries before it splits value and count: |fx| < 2^53 keeps their sum below the count field
	if (!(ws == ws) || !(v == v) || fx >= (1ll << 53) || fx <= -(1ll << 53)) atomicOr(P.bad, 2u);
	P.tval[i] = fx + ((long long)(counted ? 1 : 0) << KT_VALID_SHIFT);
}

cudaError_t run_tuple_values(const TupleValParams &P, bool recip, cudaStream_t st) {
	const unsigned g = (unsigned)(((uint64_t)P.n + 1 + 255) / 256);
	if (recip) k_tuple_values<true><<<g, 256, 0, st>>>(P);
	else k_tuple_values<false><<<g, 256, 0, st>>>(P);
	return cudaGetLastError();
}

// =================================================================== K1t
constexpr int KT_THREADS = 1024;
constexpr int KT_STEPS = 1;                       // one 16-byte + one 8-byte load in flight per thread (two steps spill at 64 registers)
constexpr int KT_GROUP = 8;                       // evaluations per thread and step
constexpr int KT_STEP_EVALS = KT_THREADS * KT_GROUP;
constexpr int KT_TILE = KT_STEP_EVALS * KT_STEPS; // 8192 evaluations

static_assert(KT_GROUP * KT_STEPS <= 16, "the count field of a table entry sits 5 bits above the largest 16-entry sum");

int kt_tile_evals() { return KT_TILE; }

// streaming loads: the index planes are read once — keep them out of L1, which serves the table tail
__device__ __forceinline__ uint4 ld_stream16(const void *p) {
	uint4 v;
	asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
	return v;
}
__device__ __forceinline__ uint2 ld_stream8(const void *p) {
	uint2 v;
	asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
	return v;
}

// table entry of index idx: shared memory below `hot`, the read-only path above — both loads predicated, no branch
__device__ __forceinline__ long long tuple_entry(uint32_t idx, uint32_t hot, uint32_t s_base, const long long *tval) {
	long long v;
	const uint32_t saddr = s_base + idx * 8u;
	const long long *g = tval + idx;
	asm("{\n\t.reg .pred p;\n\tsetp.lt.u32 p, %2, %3;\n\t@p ld.shared.s64 %0, [%1];\n\t@!p ld.global.nc.s64 %0, [%4];\n\t}"
	    : "=l"(v) : "r"(saddr), "r"(idx), "r"(hot), "l"(g));
	return v;
}

struct KtRegs { uint4 l[KT_STEPS]; uint2 h[KT_STEPS]; };

__global__ void __launch_bounds__(KT_THREADS, 1)
k_reward9t(const KtParams P) {
	extern __shared__ __align__(16) long long s_hot[];
	const int tid = threadIdx.x, lane = tid & 31;
	for (uint32_t i = tid; i < P.hot; i += KT_THREADS) s_hot[i] = P.tval[i];
	__syncthreads();
	const uint32_t s_base = smem_u32(s_hot);
	const uint32_t hot = P.hot, nclamp = P.n_tuples;               // tval[n_tuples] is the zero sentinel
	const long long *tval = P.tval;

	const uint64_t lo_t = P.total_tiles * blockIdx.x / gridDim.x;
	const uint64_t hi_t = P.total_tiles * (blockIdx.x + 1ull) / gridDim.x;
	if (lo_t >= hi_t) return;

	// (candidate, tile in row) of the tile being computed and of the one being prefetched, advanced incrementally
	uint32_t c = (uint32_t)(lo_t / P.tiles_per_cand), j = (uint32_t)(lo_t - (uint64_t)c * P.tiles_per_cand);
	uint32_t cn = c, jn = j;
	auto tile_n = [&](uint32_t jj) -> uint32_t {
		const uint64_t rem = P.T - (uint64_t)jj * KT_TILE;
		return rem < (uint64_t)KT_TILE ? (uint32_t)rem : (uint32_t)KT_TILE;
	};
	auto prefetch = [&](uint32_t cc, uint32_t jj, KtRegs &R) {
		if (tile_n(jj) != (uint32_t)KT_TILE) return;               // ragged row end: read by the scalar loop instead
		const uint64_t e0 = (uint64_t)cc * P.pitch_evals + (uint64_t)jj * KT_TILE + (uint64_t)tid * KT_GROUP;
#pragma unroll
		for (int k = 0; k < KT_STEPS; k++) {
			R.l[k] = ld_stream16(P.tl + e0 + (uint64_t)k * KT_STEP_EVALS);
			R.h[k] = ld_stream8(P.th + e0 + (uint64_t)k * KT_STEP_EVALS);
		}
	};

	Acc128 acc; acc.zero();
	uint32_t cnt = 0, seen_max = 0;
	int cur = -1;
	auto flush = [&](int cand) {
		long long *dst = P.acc + (uint64_t)ACC_PER_CAND * cand;
		flush_acc128(acc, dst, lane);
		const uint32_t n = warp_sum_u32(cnt);
		if (lane == 0 && n) atomicAdd((unsigned long long *)dst + 3, (unsigned long long)n);
		acc.zero(); cnt = 0;
	};

	KtRegs R{}, N{};
	prefetch(c, j, R);
	for (uint64_t tile = lo_t; tile < hi_t; ++tile) {
		if (++jn == P.tiles_per_cand) { jn = 0; cn++; }
		if (tile + 1 < hi_t) prefetch(cn, jn, N);
		if ((int)c != cur) { if (cur >= 0) flush(cur); cur = (int)c; }
		const uint32_t n = tile_n(j);
		if (n == (uint32_t)KT_TILE) {
			long long s = 0;
#pragma unroll
			for (int k = 0; k < KT_STEPS; k++) {
				const uint32_t lw[4] = {R.l[k].x, R.l[k].y, R.l[k].z, R.l[k].w};
				const uint32_t hw[2] = {R.h[k].x, R.h[k].y};
#pragma unroll
				for (int q = 0; q < KT_GROUP; q++) {
					// bytes {lo, hi} of the 16-bit half q&1 of word q>>1, then byte q&3 of the high-plane word q>>2
					const uint32_t sel = (q & 1 ? 0x0032u : 0x0010u) | ((4u + (q & 3)) << 8) | 0x4000u;
					uint32_t idx = __byte_perm(lw[q >> 1], hw[q >> 2], sel) & 0x00FFFFFFu;
					seen_max = max(seen_max, idx);
					idx = min(idx, nclamp);
					s += tuple_entry(idx, hot, s_base, tval);
				}
			}
			// KT_GROUP * KT_STEPS <= 16 entries: sum of values in (-2^57, 2^57) + count * 2^58
			const long long k16 = (s + (1ll << (KT_VALID_SHIFT - 1))) >> KT_VALID_SHIFT;
			acc.add(s - (k16 << KT_VALID_SHIFT));
			cnt += (uint32_t)k16;
		} else {
			const uint64_t e0 = (uint64_t)c * P.pitch_evals + (uint64_t)j * KT_TILE;
			for (uint32_t e = tid; e < n; e += KT_THREADS) {
				uint32_t idx = (uint32_t)P.tl[e0 + e] | ((uint32_t)P.th[e0 + e] << 16);
				seen_max = max(seen_max, idx);
				idx = min(idx, nclamp);
				const long long v = idx < hot ? s_hot[idx] : __ldg(tval + idx);
				const long long k1 = (v + (1ll << (KT_VALID_SHIFT - 1))) >> KT_VALID_SHIFT;
				acc.add(v - (k1 << KT_VALID_SHIFT));
				cnt += (uint32_t)k1;
			}
		}
		R = N;
		c = cn; j = jn;
	}
	if (cur >= 0) flush(cur);
	if (seen_max >= P.n_tuples) atomicOr(P.bad, 1u);
}

cudaError_t run_reward9t(KtParams P, int sm_count, cudaStream_t st) {
	P.tiles_per_cand = (uint32_t)((P.T + KT_TILE - 1) / KT_TILE);
	P.total_tiles = (uint64_t)P.tiles_per_cand * P.C;
	if (P.total_tiles == 0) return cudaSuccess;
	const uint64_t entries = (uint64_t)P.n_tuples + 1;
	P.hot = (uint32_t)(entries < KT_HOT_MAX ? entries : KT_HOT_MAX);
	const int smem = (int)(((uint64_t)P.hot * 8 + 15) & ~15ull);
	cudaError_t err = allow_big_smem(k_reward9t, (int)(KT_HOT_MAX * 8));   // set once per device: the largest head any call may ask for
	if (err != cudaSuccess) return err;
	int grid = sm_count;
	if ((uint64_t)grid > P.total_tiles) grid = (int)P.total_tiles;
	k_reward9t<<<grid, KT_THREADS, smem, st>>>(P);
	return cudaGetLastError();
}

// =================================================================== K1t2: the Form T copy from its 16-bit slot plane
// The same gather-and-add as K1t over one 16-bit plane: the registers th took carry a second 16-byte word, so each thread
// keeps 16 evaluations (32 B) in flight instead of 8 (24 B).  The plane names slots of the slot-ordered table (apo_kernels.h):
// the hot entries have one copy per shared-memory bank pair and k_slot_plane picked, per half-warp instruction, copies that
// keep clear of each other and of the single-slot lanes.  The listed evaluations (exceptions and the entries without a slot)
// read the zero slot; the CTA adds them from the entry-order table once its stream is done, four in flight per thread.
constexpr int KT2_STEPS = 2;
constexpr int KT2_TILE = KT_STEP_EVALS * KT2_STEPS;    // 16384 evaluations
constexpr int KT2_XUNROLL = 4;                         // listed evaluations in flight per thread in the correction
constexpr uint32_t KT2_HOT_MAX = 28672;                // 224 KB of shared memory: the slot-order head

static_assert(KT_GROUP * KT2_STEPS <= 16, "the count field of a table entry sits 5 bits above the largest 16-entry sum");

int kt2_tile_evals() { return KT2_TILE; }

// table entry -> (value, count)
__device__ __forceinline__ long long kt_split(long long v, int &k) {
	const long long kk = (v + (1ll << (KT_VALID_SHIFT - 1))) >> KT_VALID_SHIFT;
	k = (int)kk;
	return v - (kk << KT_VALID_SHIFT);
}

// DIAG (examples/k1t2_gather.py, builds with APO_K1T2_DIAG only): 1 adds the raw slots (the stream alone), 2 clamps the
// gather to the shared-memory head (no ld.global).  Their sums are not the table's.
template <int DIAG>
__global__ void __launch_bounds__(KT_THREADS, 1)
k_reward9t2(const Kt2Params P) {
	extern __shared__ __align__(16) long long s_hot[];
	const int tid = threadIdx.x, lane = tid & 31;
	for (uint32_t i = tid; i < P.hot; i += KT_THREADS) s_hot[i] = P.sval[i];
	__syncthreads();
	const uint32_t s_base = smem_u32(s_hot);
	const uint32_t hot = P.hot;
	const long long *sval = P.sval;

	const uint64_t lo_t = P.total_tiles * blockIdx.x / gridDim.x;
	const uint64_t hi_t = P.total_tiles * (blockIdx.x + 1ull) / gridDim.x;
	if (lo_t >= hi_t) return;

	uint32_t c = (uint32_t)(lo_t / P.tiles_per_cand), j = (uint32_t)(lo_t - (uint64_t)c * P.tiles_per_cand);
	uint32_t cn = c, jn = j;
	auto tile_n = [&](uint32_t jj) -> uint32_t {
		const uint64_t rem = P.T - (uint64_t)jj * KT2_TILE;
		return rem < (uint64_t)KT2_TILE ? (uint32_t)rem : (uint32_t)KT2_TILE;
	};
	auto prefetch = [&](uint32_t cc, uint32_t jj, uint4 (&R)[KT2_STEPS]) {
		if (tile_n(jj) != (uint32_t)KT2_TILE) return;              // ragged row end: read by the scalar loop instead
		const uint64_t e0 = (uint64_t)cc * P.pitch_evals + (uint64_t)jj * KT2_TILE + (uint64_t)tid * KT_GROUP;
#pragma unroll
		for (int k = 0; k < KT2_STEPS; k++) R[k] = ld_stream16(P.ts + e0 + (uint64_t)k * KT_STEP_EVALS);
	};
	auto entry = [&](uint32_t slot) -> long long {
		if (DIAG == 1) return (long long)slot;
		if (DIAG == 2) return s_hot[min(slot, hot - 1)];
		return tuple_entry(slot, hot, s_base, sval);
	};

	Acc128 acc; acc.zero();
	int cnt = 0;
	// the listed evaluations (list ls, block index lb) of window tiles [ja, jb) of row cc, from the entry-order table
	auto correct = [&](const uint2 *ls, const uint32_t *lb, uint32_t cc, uint32_t ja, uint32_t jb) {
		const uint64_t lo = P.first + (uint64_t)ja * KT2_TILE;
		const uint64_t hi = P.first + min((uint64_t)jb * KT2_TILE, P.T);
		const uint32_t *xr = lb + (uint64_t)cc * P.xb_pitch;
		const uint32_t x0 = xr[lo / KT_XBLOCK], x1 = xr[(hi - 1) / KT_XBLOCK + 1];   // the blocks holding [lo, hi)
		for (uint32_t x = x0 + tid; x < x1; x += KT2_XUNROLL * KT_THREADS) {
			uint32_t full[KT2_XUNROLL];
#pragma unroll
			for (int u = 0; u < KT2_XUNROLL; u++) {
				const uint32_t xi = x + u * KT_THREADS;
				const uint2 ex = xi < x1 ? __ldg(ls + xi) : make_uint2(0u, 0u);
				full[u] = xi < x1 && ex.x >= lo && ex.x < hi ? ex.y : P.n_tuples;   // the zero sentinel: no change
			}
#pragma unroll
			for (int u = 0; u < KT2_XUNROLL; u++) {
				int k;
				acc.add(kt_split(__ldg(P.tval + full[u]), k));
				cnt += k;
			}
		}
	};
	auto flush = [&](int cand) {
		long long *dst = P.acc + (uint64_t)ACC_PER_CAND * cand;
		flush_acc128(acc, dst, lane);
		const uint32_t n = warp_sum_u32((uint32_t)cnt);
		if (lane == 0 && n) atomicAdd((unsigned long long *)dst + 3, (unsigned long long)n);
		acc.zero(); cnt = 0;
	};

	uint4 R[KT2_STEPS] = {}, N[KT2_STEPS] = {};
	prefetch(c, j, R);
	int cur = -1;
	for (uint64_t tile = lo_t; tile < hi_t; ++tile) {
		if (++jn == P.tiles_per_cand) { jn = 0; cn++; }
		if (tile + 1 < hi_t) prefetch(cn, jn, N);
		if ((int)c != cur) { if (cur >= 0) flush(cur); cur = (int)c; }
		const uint32_t n = tile_n(j);
		if (n == (uint32_t)KT2_TILE) {
			long long s = 0;
#pragma unroll
			for (int k = 0; k < KT2_STEPS; k++) {
				const uint32_t lw[4] = {R[k].x, R[k].y, R[k].z, R[k].w};
#pragma unroll
				for (int q = 0; q < KT_GROUP; q++) s += entry((lw[q >> 1] >> (16 * (q & 1))) & 0xFFFFu);
			}
			int k16;
			acc.add(kt_split(s, k16));                         // 16 entries: values in (-2^57, 2^57) + count * 2^58
			cnt += k16;
		} else {
			const uint64_t e0 = (uint64_t)c * P.pitch_evals + (uint64_t)j * KT2_TILE;
			for (uint32_t e = tid; e < n; e += KT_THREADS) {
				const uint32_t slot = P.ts[e0 + e];
				int k1;
				acc.add(kt_split(DIAG ? entry(slot) : slot < hot ? s_hot[slot] : __ldg(sval + slot), k1));
				cnt += k1;
			}
		}
#pragma unroll
		for (int k = 0; k < KT2_STEPS; k++) R[k] = N[k];
		c = cn; j = jn;
	}
	flush(cur);
	// the corrections after the stream, one flush per candidate segment: inside the loop they would spill the prefetch
	if (!P.xs && !P.ys) return;
	const uint32_t c_lo = (uint32_t)(lo_t / P.tiles_per_cand), c_hi = (uint32_t)((hi_t - 1) / P.tiles_per_cand);
	for (uint32_t cc = c_lo; cc <= c_hi; cc++) {
		const uint32_t ja = cc == c_lo ? (uint32_t)(lo_t - (uint64_t)cc * P.tiles_per_cand) : 0u;
		const uint32_t jb = cc == c_hi ? (uint32_t)(hi_t - (uint64_t)cc * P.tiles_per_cand) : P.tiles_per_cand;
#pragma unroll 1
		for (int y = 0; y < 2; y++) {
			const uint2 *ls = y ? P.ys : P.xs;
			if (ls) correct(ls, y ? P.yb : P.xb, cc, ja, jb);
		}
		flush((int)cc);
	}
}

namespace {
int k1_env_grid() { static const int g = [] { const char *s = getenv("APO_K1_GRID"); return s ? atoi(s) : 0; }(); return g; }
}  // namespace

template <int DIAG>
cudaError_t launch_reward9t2(const Kt2Params &P, int grid, int smem, cudaStream_t st) {
	cudaError_t err = allow_big_smem(k_reward9t2<DIAG>, (int)(KT2_HOT_MAX * 8));   // set once per device: the largest head
	if (err != cudaSuccess) return err;
	k_reward9t2<DIAG><<<grid, KT_THREADS, smem, st>>>(P);
	return cudaGetLastError();
}

cudaError_t run_reward9t2(Kt2Params P, int sm_count, cudaStream_t st) {
	P.tiles_per_cand = (uint32_t)((P.T + KT2_TILE - 1) / KT2_TILE);
	P.total_tiles = (uint64_t)P.tiles_per_cand * P.C;
	if (P.total_tiles == 0) return cudaSuccess;
	P.hot = P.n_slots < KT2_HOT_MAX ? P.n_slots : KT2_HOT_MAX;
	const int smem = (int)(((uint64_t)P.hot * 8 + 15) & ~15ull);
	int grid = sm_count;
	if (k1_env_grid() > 0 && k1_env_grid() < grid) grid = k1_env_grid();   // tests: every CTA cut of the rows and the lists
	if ((uint64_t)grid > P.total_tiles) grid = (int)P.total_tiles;
#ifdef APO_K1T2_DIAG
	const char *d = getenv("APO_K1T2_DIAG");                    // read per launch: one process alternates the variants
	if (d && atoi(d) == 1) return launch_reward9t2<1>(P, grid, smem, st);
	if (d && atoi(d) == 2) return launch_reward9t2<2>(P, grid, smem, st);
#endif
	return launch_reward9t2<0>(P, grid, smem, st);
}

// =================================================================== K1h: whole rows of the Form T copy from its counts
// Each CTA takes a contiguous range of the pair array (the rows' pairs back to back), finds its first row by a search of the
// offsets and walks the rows the range covers; every warp flushes once per row.  Per pair: one 8-byte load, the entry's table
// value through the read-only path (a row's entries ascend, so a warp's gathers land in neighbouring sectors) and the exact
// 128-bit count * value.  With the corpus report the CTA's last warp runs its share of the digest pass meanwhile (cd_warp), so
// only the ticket and the finalisation follow the stream.  One warp takes ~90 ns per digest entry where the CTA's stream takes
// ~0.45 ns per pair (H100, DESIGN §8).  A CTA with fewer than KH_PAIRS_PER_ENTRY pairs per entry of its digest share (small C
// or T), whose lone digest warp would outlast its stream by more than the block-wide pass costs after it, streams on all 32
// warps and then runs the pass block-wide, as the stand-alone k_corpus_digest does.  The flagship has ~215 pairs per entry.
constexpr int KH_THREADS = 1024;
constexpr int KH_UNROLL = 8;                      // pairs in flight per thread
constexpr uint64_t KH_PAIRS_PER_ENTRY = 128;

#ifdef APO_K1H_DIAG
// examples/flagship_launch.py: the phases of every CTA as %globaltimer stamps (kh_stamp, apo_corpus.cuh), and with
// APO_K1H_DIAG=1 the stream alone: the gather replaced by a constant (its sums are not the table's)
extern "C" int apo_diag_k1h_stamps(unsigned long long *out, uint32_t n) {
	cudaError_t err = cudaMemcpyFromSymbol(out, g_kh_stamp, sizeof(unsigned long long) * (n < KH_STAMP_WORDS ? n : KH_STAMP_WORDS));
	void *p = nullptr;
	if (err == cudaSuccess) err = cudaGetSymbolAddress(&p, g_kh_stamp);
	if (err == cudaSuccess) err = cudaMemset(p, 0, sizeof(g_kh_stamp));
	return (int)err;
}
#endif

// the rows of pairs [lo, hi) of one CTA, streamed by its first NT threads
template <int NT, int DIAG>
__device__ __forceinline__ void kh_rows(const KhParams &P, uint64_t lo, uint64_t hi, int tid, int lane) {
	uint32_t a = 0, b = P.C;                                       // off[a] <= lo < off[b]: 32 offsets per step, not 2
	while (b - a > 1) {
		const uint32_t step = (b - a + 31) / 32, i = a + (uint32_t)lane * step;
		const unsigned le = __ballot_sync(0xffffffffu, i < b && P.off[i] <= lo);     // lane 0 (off[a]) always; the rest ascend
		a += (31u - __clz(le)) * step;
		b = min(a + step, b);
	}
	for (uint32_t c = a; c < P.C; c++) {
		const uint64_t r0 = P.off[c], r1 = P.off[c + 1];
		if (r0 >= hi) break;
		const uint64_t s = max(lo, r0), t = min(hi, r1);
		Acc128 acc; acc.zero();
		unsigned long long cnt = 0;
		for (uint64_t p = s + tid; p < t; p += (uint64_t)NT * KH_UNROLL) {
			unsigned long long w[KH_UNROLL];
#pragma unroll
			for (int u = 0; u < KH_UNROLL; u++) {
				const uint64_t q = p + (uint64_t)u * NT;
				if (q < t) { const uint2 v = ld_stream8(P.pairs + q); w[u] = (unsigned long long)v.x | ((unsigned long long)v.y << 32); }
				else w[u] = 0;                                        // entry 0, count 0: adds nothing
			}
#pragma unroll
			for (int u = 0; u < KH_UNROLL; u++) {
				const unsigned long long n = w[u] >> KH_COUNT_SHIFT;
				const uint32_t entry = (uint32_t)(w[u] & ((1u << KH_COUNT_SHIFT) - 1u));
				int k;
				const long long v = kt_split(DIAG ? (1ll << KT_VALID_SHIFT) + entry : __ldg(P.tval + entry), k);
				acc_add_mul(acc, n, v);
				cnt += k ? n : 0ull;
			}
		}
		if (s >= t) continue;
		long long *dst = P.acc + (uint64_t)ACC_PER_CAND * c;
		flush_acc128(acc, dst, lane);
		const unsigned long long nc = warp_sum_u64(cnt);
		if (lane == 0 && nc) atomicAdd((unsigned long long *)dst + 3, nc);
	}
}

template <int DIAG>
__global__ void __launch_bounds__(KH_THREADS, 1)
k_reward9th(const __grid_constant__ KhParams P) {      // grid constant: the digest pass reads P.cd in place, no per-thread copy
	const int tid = threadIdx.x, lane = tid & 31;
	kh_stamp(KH_ST_ENTRY);
	const uint64_t lo = P.nnz * blockIdx.x / gridDim.x, hi = P.nnz * (blockIdx.x + 1ull) / gridDim.x;
	if (!P.corpus_on) {
		if (lo < hi) kh_rows<KH_THREADS, DIAG>(P, lo, hi, tid, lane);
		return;
	}
	const uint64_t share = P.cd_n * (blockIdx.x + 1ull) / gridDim.x - P.cd_n * blockIdx.x / gridDim.x;   // block-uniform
	if (hi - lo < KH_PAIRS_PER_ENTRY * share) {                        // the digest share outlasts the pairs: all warps on both
		if (lo < hi) kh_rows<KH_THREADS, DIAG>(P, lo, hi, tid, lane);
		kh_stamp_max(KH_ST_PAIRS);
		corpus_digest_block(P.cd);
		return;
	}
	if (tid >= KH_THREADS - 32) {                                      // the last warp: this CTA's share of the digest
		cd_warp(P.cd);
		kh_stamp_max(KH_ST_DIGEST);
	} else {
		if (lo < hi) kh_rows<KH_THREADS - 32, DIAG>(P, lo, hi, tid, lane);
		kh_stamp_max(KH_ST_PAIRS);
	}
	cd_tail(P.cd, cd_shared());                                        // every CTA, with or without pairs: block-wide
}

cudaError_t run_reward9th(const KhParams &P, int sm_count, cudaStream_t st) {
	if (P.nnz == 0 && !P.corpus_on) return cudaSuccess;
	int grid = sm_count;
	if (k1_env_grid() > 0 && k1_env_grid() < grid) grid = k1_env_grid();   // tests: every CTA cut of the rows
	const uint64_t need = (P.nnz + KH_THREADS - 1) / KH_THREADS;
	if ((uint64_t)grid > need) grid = (int)need;
	if (grid < 1) grid = 1;                                                  // no pairs: one CTA for the corpus words and the tail
#ifdef APO_K1H_DIAG
	if (const char *d = getenv("APO_K1H_DIAG"); d && atoi(d) == 1) {       // read per launch: one process alternates the variants
		k_reward9th<1><<<grid, KH_THREADS, 0, st>>>(P);
		return cudaGetLastError();
	}
#endif
	k_reward9th<0><<<grid, KH_THREADS, 0, st>>>(P);
	return cudaGetLastError();
}

// ---- the counts, built at load: a count pass into a dense [rows][npitch] scratch, then per (row, chunk of TH_CHUNK entries)
// a count of the non-zero entries, one exclusive scan, and an ordered write
constexpr int TH_THREADS = 256;
constexpr uint32_t TH_CHUNK = TH_THREADS * 32;    // 32 entries per thread

__global__ void __launch_bounds__(1024) k_tx_scan(uint32_t *xb, uint64_t n);   // the lists' scan, below

__global__ void __launch_bounds__(256)
k_th_count(const unsigned short *tl, const unsigned char *th, uint64_t tpitch, uint32_t R, uint64_t T, uint32_t npitch, uint32_t *cnt) {
	const uint32_t lane = threadIdx.x & 31;
	const uint64_t gpr = (T + 7) / 8, groups = (uint64_t)R * gpr;
	// the loop bound is block-uniform: match.any needs every lane
	for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < groups; base += (uint64_t)gridDim.x * blockDim.x) {
		const uint64_t g = base + threadIdx.x;
		uint64_t r = 0, t0 = T;
		uint4 l = make_uint4(0u, 0u, 0u, 0u);
		uint2 h = make_uint2(0u, 0u);
		if (g < groups) {
			r = g / gpr; t0 = (g - r * gpr) * 8;
			l = ld_stream16(tl + r * tpitch + t0);
			h = ld_stream8(th + r * tpitch + t0);
		}
		const uint32_t lw[4] = {l.x, l.y, l.z, l.w}, hw[2] = {h.x, h.y};
#pragma unroll
		for (int q = 0; q < 8; q++) {
			const uint32_t sel = (q & 1 ? 0x0032u : 0x0010u) | ((4u + (q & 3)) << 8) | 0x4000u;   // as K1t
			const uint32_t idx = __byte_perm(lw[q >> 1], hw[q >> 2], sel) & 0x00FFFFFFu;
			const bool valid = t0 + q < T;                            // pads are not counted
			const unsigned long long key = valid ? r * npitch + idx : ~0ull;
			const uint32_t peers = __match_any_sync(0xFFFFFFFFu, key);
			if (valid && (uint32_t)(__ffs(peers) - 1) == lane) atomicAdd(cnt + key, (uint32_t)__popc(peers));
		}
	}
}

// WRITE = false: nz[it] = the non-zero entries of item it = (row, chunk), and nz[R * nchunk] = 0 (the scan makes it the total).
// WRITE: their pairs, from base + nz[it] on (nz scanned), and the row offsets.
template <bool WRITE>
__global__ void __launch_bounds__(TH_THREADS)
k_th_rows(const uint32_t *cnt, uint32_t R, uint32_t npitch, uint32_t nchunk, uint32_t *nz, uint64_t base, unsigned long long *pairs,
          uint64_t *off) {
	__shared__ uint32_t s_w[TH_THREADS / 32];
	const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint64_t items = (uint64_t)R * nchunk;
	for (uint64_t it = blockIdx.x; it < items; it += gridDim.x) {
		const uint32_t r = (uint32_t)(it / nchunk), b = (uint32_t)(it - (uint64_t)r * nchunk);
		const uint32_t e0 = b * TH_CHUNK + threadIdx.x * 32;
		uint32_t v[32], m = 0;
#pragma unroll
		for (int i = 0; i < 8; i++) {
			const uint4 x = e0 < npitch ? *reinterpret_cast<const uint4 *>(cnt + (uint64_t)r * npitch + e0 + 4 * i) : make_uint4(0u, 0u, 0u, 0u);
			v[4 * i] = x.x; v[4 * i + 1] = x.y; v[4 * i + 2] = x.z; v[4 * i + 3] = x.w;
		}
#pragma unroll
		for (int q = 0; q < 32; q++) m |= (v[q] ? 1u : 0u) << q;
		const uint32_t k = (uint32_t)__popc(m);
		if (!WRITE) {
			const uint32_t s = warp_sum_u32(k);
			if (lane == 0) s_w[warp] = s;
			__syncthreads();
			if (threadIdx.x == 0) {
				uint32_t t = 0;
				for (int w = 0; w < TH_THREADS / 32; w++) t += s_w[w];
				nz[it] = t;
				if (it == items - 1) nz[items] = 0;
			}
			__syncthreads();
			continue;
		}
		uint32_t incl = k;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) { const uint32_t x = __shfl_up_sync(0xFFFFFFFFu, incl, o); if (lane >= (uint32_t)o) incl += x; }
		if (lane == 31) s_w[warp] = incl;
		__syncthreads();
		uint64_t o = base + nz[it] + incl - k;
		for (uint32_t w = 0; w < warp; w++) o += s_w[w];
		if (threadIdx.x == 0 && b == 0) off[r] = base + nz[it];
		if (threadIdx.x == 0 && it == items - 1) off[R] = base + nz[items];
#pragma unroll
		for (int q = 0; q < 32; q++)
			if ((m >> q) & 1u) pairs[o++] = (unsigned long long)(e0 + q) | ((unsigned long long)v[q] << KH_COUNT_SHIFT);
		__syncthreads();
	}
}

namespace {
unsigned th_grid(uint64_t items, int sm_count) { return (unsigned)(items < 8ull * sm_count ? items : 8ull * sm_count); }
}  // namespace

cudaError_t run_th_count(const unsigned short *tl, const unsigned char *th, uint64_t tpitch, uint32_t R, uint64_t T, uint32_t npitch,
                         uint32_t *cnt, uint32_t *nz, int sm_count, cudaStream_t st) {
	const uint64_t groups = (uint64_t)R * ((T + 7) / 8);
	const uint32_t nchunk = (npitch + TH_CHUNK - 1) / TH_CHUNK;
	if (groups == 0 || nchunk == 0) return cudaSuccess;
	k_th_count<<<th_grid((groups + 255) / 256, sm_count), 256, 0, st>>>(tl, th, tpitch, R, T, npitch, cnt);
	const uint64_t items = (uint64_t)R * nchunk;
	k_th_rows<false><<<th_grid(items, sm_count), TH_THREADS, 0, st>>>(cnt, R, npitch, nchunk, nz, 0, nullptr, nullptr);
	k_tx_scan<<<1, 1024, 0, st>>>(nz, items + 1);
	return cudaGetLastError();
}

cudaError_t run_th_write(const uint32_t *cnt, uint32_t R, uint32_t npitch, const uint32_t *nz, uint64_t base, unsigned long long *pairs,
                         uint64_t *off, int sm_count, cudaStream_t st) {
	const uint32_t nchunk = (npitch + TH_CHUNK - 1) / TH_CHUNK;
	const uint64_t items = (uint64_t)R * nchunk;
	if (items == 0) return cudaSuccess;
	k_th_rows<true><<<th_grid(items, sm_count), TH_THREADS, 0, st>>>(cnt, R, npitch, nchunk, const_cast<uint32_t *>(nz), base, pairs, off);
	return cudaGetLastError();
}

// ---- the slot-order table and the slot plane (apo_kernels.h)
__global__ void __launch_bounds__(256)
k_tuple_slots(const long long *tval, uint32_t h, uint32_t end, long long *sval) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, z = KT_SLOT_REP * h;
	if (i > end + (KT_SLOT_REP - 1) * h) return;
	sval[i] = i < z ? tval[i / KT_SLOT_REP] : i == z ? 0ll : tval[i - (KT_SLOT_REP - 1) * h - 1];
}

cudaError_t run_tuple_slots(const long long *tval, uint32_t h, uint32_t end, long long *sval, cudaStream_t st) {
	const uint32_t n = end + (KT_SLOT_REP - 1) * h + 1;
	k_tuple_slots<<<(n + 255) / 256, 256, 0, st>>>(tval, h, end, sval);
	return cudaGetLastError();
}

// One thread per half-warp instruction of K1t2 on a window that starts on the 128-evaluation grid: evaluations
// b * 128 + 8 l + q, l < 16, of a row.  The single-slot lanes (and the zero slot) claim their bank pairs first; each distinct
// hot entry then takes the copy in its own lane's bank pair if that is free, else the lowest free one (equal entries share a
// copy: a broadcast).  When more distinct addresses meet than there are bank pairs the conflict cannot be avoided anyway.
__global__ void __launch_bounds__(256)
k_slot_plane(const unsigned short *tl, const unsigned char *th, uint64_t tpitch, uint32_t C, uint64_t T, uint32_t h, uint32_t end,
             unsigned short *ts) {
	const uint64_t nb = (T + 127) / 128, items = (uint64_t)C * nb * 8;
	for (uint64_t it = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; it < items; it += (uint64_t)gridDim.x * blockDim.x) {
		const uint32_t q = (uint32_t)(it & 7u);
		const uint64_t r = it >> 3, c = r / nb, b = r - c * nb;
		const uint64_t row = c * tpitch, t0 = b * 128 + q;
		uint32_t e[16], used = 0, hot = 0;
#pragma unroll
		for (int l = 0; l < 16; l++) {
			const uint64_t t = t0 + 8 * l;
			e[l] = t < T ? (uint32_t)tl[row + t] | ((uint32_t)th[row + t] << 16) : 0xFFFFFFFFu;
			if (e[l] < h) hot |= 1u << l;
			else if (t < T) used |= 1u << ((e[l] < end ? e[l] + (KT_SLOT_REP - 1) * h + 1 : KT_SLOT_REP * h) & 15u);
		}
		uint32_t bp[16];
#pragma unroll
		for (int l = 0; l < 16; l++) {
			bp[l] = 16;
			if (!((hot >> l) & 1u)) continue;
#pragma unroll
			for (int m = 0; m < l; m++)
				if (bp[l] == 16 && ((hot >> m) & 1u) && e[m] == e[l]) bp[l] = bp[m];
			if (bp[l] == 16) {
				const uint32_t free = ~used & 0xFFFFu;
				bp[l] = ((free >> l) & 1u) || !free ? (uint32_t)l : (uint32_t)(__ffs(free) - 1);
				used |= 1u << bp[l];
			}
		}
#pragma unroll
		for (int l = 0; l < 16; l++) {
			const uint64_t t = t0 + 8 * l;
			if (t >= T) continue;
			const uint32_t s = (hot >> l) & 1u ? KT_SLOT_REP * e[l] + bp[l] : e[l] < end ? e[l] + (KT_SLOT_REP - 1) * h + 1 : KT_SLOT_REP * h;
			ts[row + t] = (unsigned short)s;
		}
	}
}

cudaError_t run_slot_plane(const unsigned short *tl, const unsigned char *th, uint64_t tpitch, uint32_t C, uint64_t T, uint32_t h,
                           uint32_t end, unsigned short *ts, cudaStream_t st) {
	const uint64_t items = (uint64_t)C * ((T + 127) / 128) * 8;
	if (items == 0) return cudaSuccess;
	uint64_t g = (items + 255) / 256;
	if (g > 132ull * 64) g = 132ull * 64;
	k_slot_plane<<<(unsigned)g, 256, 0, st>>>(tl, th, tpitch, C, T, h, end, ts);
	return cudaGetLastError();
}

// ---- the lists, built on the device from the planes: a count pass per (row, block), one exclusive scan over [C][nblk + 1],
// and an ordered write pass.  Each (row, block) is one CTA's item, 32 evaluations per thread.  LOW: the evaluations whose
// index is in [lo, 2^16) instead of the exceptions.
constexpr int TX_THREADS = 256;
constexpr int TX_EVALS = KT_XBLOCK / TX_THREADS;       // 32
static_assert(TX_EVALS == 32, "one bit per evaluation of a thread");

// bit q: evaluation t0 + q (< T) of the row has a non-zero high byte (LOW: a zero high byte and a low half >= lo)
template <bool LOW>
__device__ __forceinline__ uint32_t tx_mask(const unsigned short *tl_row, const unsigned char *th_row, uint64_t t0, uint64_t T, uint32_t lo) {
	if (t0 >= T) return 0u;
	const uint4 a = ld_stream16(th_row + t0), b = ld_stream16(th_row + t0 + 16);   // inside the row's 64-padded pitch
	const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
	uint32_t m = 0;
	if (LOW) {
#pragma unroll
		for (int i = 0; i < 4; i++) {
			const uint4 v = ld_stream16(tl_row + t0 + 8 * i);
			const uint32_t lw[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
			for (int u = 0; u < 8; u++) {
				const int q = 8 * i + u;
				const bool in = ((w[q >> 2] >> (8 * (q & 3))) & 0xFFu) == 0u && ((lw[u >> 1] >> (16 * (u & 1))) & 0xFFFFu) >= lo;
				m |= (in ? 1u : 0u) << q;
			}
		}
	} else {
#pragma unroll
		for (int q = 0; q < 32; q++) m |= (((w[q >> 2] >> (8 * (q & 3))) & 0xFFu) != 0u ? 1u : 0u) << q;
	}
	const uint64_t left = T - t0;
	return left >= 32 ? m : m & ((1u << left) - 1u);
}

template <bool LOW>
__global__ void __launch_bounds__(TX_THREADS)
k_tx_count(const unsigned short *tl, const unsigned char *th, uint64_t tpitch, uint32_t C, uint64_t T, uint32_t lo, uint32_t nblk, uint32_t *xb) {
	__shared__ uint32_t s_w[TX_THREADS / 32];
	const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	for (uint64_t it = blockIdx.x; it < (uint64_t)C * nblk; it += gridDim.x) {
		const uint32_t c = (uint32_t)(it / nblk), b = (uint32_t)(it - (uint64_t)c * nblk);
		const uint32_t n = warp_sum_u32((uint32_t)__popc(tx_mask<LOW>(tl + (uint64_t)c * tpitch, th + (uint64_t)c * tpitch, (uint64_t)b * KT_XBLOCK + threadIdx.x * TX_EVALS, T, lo)));
		if (lane == 0) s_w[warp] = n;
		__syncthreads();
		if (threadIdx.x == 0) {
			uint32_t s = 0;
			for (int w = 0; w < TX_THREADS / 32; w++) s += s_w[w];
			xb[(uint64_t)c * (nblk + 1) + b] = s;
			if (b == nblk - 1) xb[(uint64_t)c * (nblk + 1) + nblk] = 0;
		}
		__syncthreads();
	}
}

// exclusive scan of xb[0, n) in place, one CTA: each thread a contiguous run
__global__ void __launch_bounds__(1024)
k_tx_scan(uint32_t *xb, uint64_t n) {
	__shared__ uint32_t s_w[32];
	const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint64_t per = (n + 1023) / 1024, lo = min(n, (uint64_t)threadIdx.x * per), hi = min(n, lo + per);
	uint32_t s = 0;
	for (uint64_t i = lo; i < hi; i++) s += xb[i];
	uint32_t incl = s;
#pragma unroll
	for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, incl, o); if (lane >= (uint32_t)o) incl += v; }
	if (lane == 31) s_w[warp] = incl;
	__syncthreads();
	if (warp == 0) {
		uint32_t w = s_w[lane];
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, w, o); if (lane >= (uint32_t)o) w += v; }
		s_w[lane] = w;
	}
	__syncthreads();
	uint32_t run = (warp ? s_w[warp - 1] : 0u) + incl - s;
	for (uint64_t i = lo; i < hi; i++) { const uint32_t v = xb[i]; xb[i] = run; run += v; }
}

template <bool LOW>
__global__ void __launch_bounds__(TX_THREADS)
k_tx_write(const unsigned short *tl, const unsigned char *th, uint64_t tpitch, uint32_t C, uint64_t T, uint32_t lo, uint32_t nblk, const uint32_t *xb,
           uint2 *xs) {
	__shared__ uint32_t s_w[TX_THREADS / 32];
	const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	for (uint64_t it = blockIdx.x; it < (uint64_t)C * nblk; it += gridDim.x) {
		const uint32_t c = (uint32_t)(it / nblk), b = (uint32_t)(it - (uint64_t)c * nblk);
		const uint64_t t0 = (uint64_t)b * KT_XBLOCK + threadIdx.x * TX_EVALS;
		uint32_t m = tx_mask<LOW>(tl + (uint64_t)c * tpitch, th + (uint64_t)c * tpitch, t0, T, lo);
		const uint32_t n = (uint32_t)__popc(m);
		uint32_t incl = n;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xFFFFFFFFu, incl, o); if (lane >= (uint32_t)o) incl += v; }
		if (lane == 31) s_w[warp] = incl;
		__syncthreads();
		uint32_t o = xb[(uint64_t)c * (nblk + 1) + b] + incl - n;
		for (uint32_t w = 0; w < warp; w++) o += s_w[w];
		while (m) {
			const uint32_t q = (uint32_t)(__ffs(m) - 1);
			m &= m - 1;
			const uint64_t t = t0 + q, off = (uint64_t)c * tpitch + t;
			xs[o++] = make_uint2((uint32_t)t, (uint32_t)tl[off] | ((uint32_t)th[off] << 16));
		}
		__syncthreads();
	}
}

cudaError_t run_tx_build(const unsigned short *tl, const unsigned char *th, uint64_t tpitch, uint32_t C, uint64_t T, uint32_t lo,
                         uint32_t *xb, uint2 *xs, int sm_count, cudaStream_t st) {
	const uint32_t nblk = (uint32_t)((T + KT_XBLOCK - 1) / KT_XBLOCK);
	const uint64_t items = (uint64_t)C * nblk;
	if (items == 0) return cudaSuccess;
	uint64_t grid = 8ull * (uint64_t)sm_count;
	if (k1_env_grid() > 0 && (uint64_t)k1_env_grid() < grid) grid = (uint64_t)k1_env_grid();
	if (grid > items) grid = items;
	const bool low = lo < 65536u;
	if (low) k_tx_count<true><<<(unsigned)grid, TX_THREADS, 0, st>>>(tl, th, tpitch, C, T, lo, nblk, xb);
	else k_tx_count<false><<<(unsigned)grid, TX_THREADS, 0, st>>>(tl, th, tpitch, C, T, lo, nblk, xb);
	k_tx_scan<<<1, 1024, 0, st>>>(xb, (uint64_t)C * (nblk + 1));
	if (low) k_tx_write<true><<<(unsigned)grid, TX_THREADS, 0, st>>>(tl, th, tpitch, C, T, lo, nblk, xb, xs);
	else k_tx_write<false><<<(unsigned)grid, TX_THREADS, 0, st>>>(tl, th, tpitch, C, T, lo, nblk, xb, xs);
	return cudaGetLastError();
}

// =================================================================== Form T built on the device (apo_dims_tuples)
// Two passes over the resident evaluations, 8 per thread and step (one row segment of 64 B of Form W):
//   count: exact counts of the distinct keys.  A warp first merges equal keys (match.any), then each CTA adds them into its
//          own shared-memory table; a key that finds no room there (the CTA met more distinct keys than the table holds: the
//          cold tail of the distribution) goes straight to the global table.  Generated data is heavily skewed, so nearly
//          every evaluation ends in a shared-memory atomic and the global table sees one add per CTA and hot key.
//   index: the rank of every evaluation's key, the hot head of the dictionary from a shared-memory table, the tail from the
//          global one (which holds only the dictionary's entries, so it stays in L2), written as Form T's tl / th.
// The dictionary order (count desc, key asc) is decided on the host from the exact counts: every grid gives the same bytes.
constexpr int TB_THREADS = 512;
constexpr int TB_GROUP = 8;                       // evaluations per thread and step
constexpr uint32_t TB_CSLOTS = 8192;              // count pass: per-CTA table, 96 KB (8-byte keys, 4-byte counts)
constexpr int TB_CPROBES = 8;                     // probes before a key goes to the global table
constexpr uint32_t TB_ISLOTS = 8192;              // index pass: per-CTA table of the hot head, 96 KB
constexpr uint32_t TB_IHOT = TB_ISLOTS / 2;       // dictionary entries in it (load 0.5: a miss ends after ~2.5 probes)

__device__ __forceinline__ uint32_t tb_hash(unsigned long long k) {
	uint32_t h = (uint32_t)k * 0x9E3779B1u ^ (uint32_t)(k >> 32) * 0x85EBCA77u;
	h ^= h >> 15; h *= 0x2C1B3C6Du; h ^= h >> 12;
	return h;
}
__device__ __forceinline__ uint32_t tb_shash(uint32_t h) { return (h * 0x9E3779B1u) >> 19; }   // 13 bits, independent of the low ones

// keys of the 8 evaluations [t0, t0 + 8) of row c; bit q of the result set when t0 + q < T
__device__ __forceinline__ uint32_t tb_keys(const TbSource &S, uint32_t c, uint64_t t0, unsigned long long k[TB_GROUP]) {
	const uint64_t off = (uint64_t)c * S.pitch + t0;
	if (S.qw) {
#pragma unroll
		for (int i = 0; i < TB_GROUP / 2; i++) {
			const uint4 v = ld_stream16(S.qw + off + 2 * i);
			k[2 * i] = (unsigned long long)v.x | ((unsigned long long)v.y << 32);
			k[2 * i + 1] = (unsigned long long)v.z | ((unsigned long long)v.w << 32);
		}
	} else {
		// k_pack_p's arithmetic: codes < 15 (checked on the host) and 255 = absent -> nibble 15; dimension 2 is bit 6 of li
		const uint4 lv = ld_stream16(S.li + off);
		const uint32_t lw[4] = {lv.x, lv.y, lv.z, lv.w};
#pragma unroll
		for (int h = 0; h < 2; h++) {
			const uint4 dv = ld_stream16(S.d2 + off + 4 * h);
			const uint32_t dw[4] = {dv.x, dv.y, dv.z, dv.w};
#pragma unroll
			for (int i = 0; i < 2; i++) {
				const uint4 qv = ld_stream16(S.q8 + off + 4 * h + 2 * i);
				const uint32_t qw[4] = {qv.x, qv.y, qv.z, qv.w};
#pragma unroll
				for (int e = 0; e < 2; e++) {
					const int q = 4 * h + 2 * i + e;
					uint32_t a = qw[2 * e] & 0x0F0F0F0Fu, b = qw[2 * e + 1] & 0x0F0F0F0Fu;
					a = (a | (a >> 4)) & 0x00FF00FFu; a = (a | (a >> 8)) & 0xFFFFu;
					b = (b | (b >> 4)) & 0x00FF00FFu; b = (b | (b >> 8)) & 0xFFFFu;
					const uint32_t li = (lw[q >> 1] >> (16 * (q & 1))) & 0xFFFFu;
					const uint32_t d = ((li >> 6) & 1u) ? dw[2 * i + e] : KW_D2_ABSENT;
					k[q] = (unsigned long long)(a | (b << 16)) | ((unsigned long long)d << 32);
				}
			}
		}
	}
	const uint64_t left = S.T - t0;
	return left >= (uint64_t)TB_GROUP ? 0xFFu : (1u << left) - 1u;
}

__device__ __forceinline__ void tb_global_add(unsigned long long *table, uint32_t mask, unsigned long long k, unsigned long long n,
                                              uint64_t cap, unsigned long long *nkeys, uint32_t *over) {
	uint32_t h = tb_hash(k) & mask;
	for (uint32_t p = 0; p <= mask; p++) {
		unsigned long long *slot = table + 2ull * h;
		unsigned long long cur = *(volatile unsigned long long *)slot;
		if (cur == TB_EMPTY) {
			cur = atomicCAS(slot, TB_EMPTY, k);
			if (cur == TB_EMPTY) {
				if (atomicAdd(nkeys, 1ull) + 1 > cap) atomicOr(over, 1u);
				cur = k;
			}
		}
		if (cur == k) { atomicAdd(slot + 1, n); return; }
		h = (h + 1) & mask;
	}
	atomicOr(over, 1u);                           // the table is full: it holds more than cap keys
}

__global__ void __launch_bounds__(256)
k_tb_clear(unsigned long long *table, uint64_t slots) {
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < slots; i += (uint64_t)gridDim.x * blockDim.x)
		reinterpret_cast<ulonglong2 *>(table)[i] = make_ulonglong2(TB_EMPTY, 0ull);
}

__global__ void __launch_bounds__(TB_THREADS, 2)
k_tb_count(const TbSource S, unsigned long long *table, uint32_t mask, uint64_t cap, unsigned long long *nkeys, uint32_t *over) {
	extern __shared__ __align__(16) unsigned long long s_tb[];
	// 32-bit counts (a native shared-memory add; the 64-bit one is a CAS loop): run_tb_count gives no CTA 2^32 evaluations
	unsigned long long *s_key = s_tb;
	uint32_t *s_cnt = reinterpret_cast<uint32_t *>(s_tb + TB_CSLOTS);
	for (uint32_t i = threadIdx.x; i < TB_CSLOTS; i += TB_THREADS) { s_key[i] = TB_EMPTY; s_cnt[i] = 0; }
	__syncthreads();
	const uint32_t lane = threadIdx.x & 31;
	const uint64_t gpr = (S.T + TB_GROUP - 1) / TB_GROUP, groups = (uint64_t)S.C * gpr;
	// the loop bound is warp-uniform (match.any and the early stop need every lane)
	for (uint64_t base = (uint64_t)blockIdx.x * TB_THREADS; base < groups; base += (uint64_t)gridDim.x * TB_THREADS) {
		const uint32_t stop = lane == 0 ? *(volatile uint32_t *)over : 0u;
		if (__any_sync(0xFFFFFFFFu, stop)) break;           // more than cap keys: the call fails, the counts are not needed
		const uint64_t g = base + threadIdx.x;
		unsigned long long k[TB_GROUP];
		uint32_t valid = 0;
		if (g < groups) {
			const uint32_t c = (uint32_t)(g / gpr);
			valid = tb_keys(S, c, (g - (uint64_t)c * gpr) * TB_GROUP, k);
		}
#pragma unroll
		for (int q = 0; q < TB_GROUP; q++) {
			const unsigned long long key = (valid >> q) & 1u ? k[q] : TB_EMPTY;
			const uint32_t peers = __match_any_sync(0xFFFFFFFFu, key);
			if (key == TB_EMPTY || (uint32_t)(__ffs(peers) - 1) != lane) continue;
			const uint32_t n = (uint32_t)__popc(peers);
			const uint32_t h0 = tb_hash(key);
			uint32_t h = tb_shash(h0) & (TB_CSLOTS - 1);
			bool done = false;
			for (int p = 0; p < TB_CPROBES; p++) {
				unsigned long long cur = *(volatile unsigned long long *)&s_key[h];
				if (cur == TB_EMPTY) {
					cur = atomicCAS(&s_key[h], TB_EMPTY, key);
					if (cur == TB_EMPTY) cur = key;
				}
				if (cur == key) { atomicAdd(&s_cnt[h], n); done = true; break; }
				h = (h + 1) & (TB_CSLOTS - 1);
			}
			if (!done) tb_global_add(table, mask, key, n, cap, nkeys, over);
		}
	}
	__syncthreads();
	for (uint32_t i = threadIdx.x; i < TB_CSLOTS; i += TB_THREADS)
		if (s_key[i] != TB_EMPTY) tb_global_add(table, mask, s_key[i], s_cnt[i], cap, nkeys, over);
}

__global__ void __launch_bounds__(256)
k_tb_compact(const unsigned long long *table, uint64_t slots, unsigned long long *keys, unsigned long long *counts, unsigned long long *n) {
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < slots; i += (uint64_t)gridDim.x * blockDim.x) {
		const ulonglong2 v = reinterpret_cast<const ulonglong2 *>(table)[i];
		if (v.x == TB_EMPTY) continue;
		const unsigned long long o = atomicAdd(n, 1ull);
		keys[o] = v.x; counts[o] = v.y;
	}
}

__global__ void __launch_bounds__(256)
k_tb_insert(const unsigned long long *keys, uint32_t n, unsigned long long *table, uint32_t mask) {
	const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
	if (r >= n) return;
	const unsigned long long k = keys[r];
	uint32_t h = tb_hash(k) & mask;
	while (atomicCAS(table + 2ull * h, TB_EMPTY, k) != TB_EMPTY) h = (h + 1) & mask;   // keys are distinct, slots >= 2 n
	table[2ull * h + 1] = r;
}

__global__ void __launch_bounds__(TB_THREADS, 2)
k_tb_index(const TbSource S, const unsigned long long *keys, uint32_t n, const unsigned long long *table, uint32_t mask,
           unsigned short *tl, unsigned char *th, uint64_t tpitch, uint32_t *bad) {
	extern __shared__ __align__(16) unsigned long long s_tb[];
	unsigned long long *s_key = s_tb;
	uint32_t *s_rank = reinterpret_cast<uint32_t *>(s_tb + TB_ISLOTS);
	for (uint32_t i = threadIdx.x; i < TB_ISLOTS; i += TB_THREADS) s_key[i] = TB_EMPTY;
	__syncthreads();
	const uint32_t hot = n < TB_IHOT ? n : TB_IHOT;
	for (uint32_t r = threadIdx.x; r < hot; r += TB_THREADS) {
		const unsigned long long k = keys[r];
		uint32_t h = tb_shash(tb_hash(k)) & (TB_ISLOTS - 1);
		while (atomicCAS(&s_key[h], TB_EMPTY, k) != TB_EMPTY) h = (h + 1) & (TB_ISLOTS - 1);
		s_rank[h] = r;
	}
	__syncthreads();
	bool missing = false;
	const uint64_t gpr = (S.T + TB_GROUP - 1) / TB_GROUP, groups = (uint64_t)S.C * gpr;
	for (uint64_t g = (uint64_t)blockIdx.x * TB_THREADS + threadIdx.x; g < groups; g += (uint64_t)gridDim.x * TB_THREADS) {
		const uint32_t c = (uint32_t)(g / gpr);
		const uint64_t t0 = (g - (uint64_t)c * gpr) * TB_GROUP;
		unsigned long long k[TB_GROUP];
		const uint32_t valid = tb_keys(S, c, t0, k);
		uint32_t lo[TB_GROUP / 2] = {0, 0, 0, 0}, hi[TB_GROUP / 4] = {0, 0};
#pragma unroll
		for (int q = 0; q < TB_GROUP; q++) {
			uint32_t r = 0;
			if ((valid >> q) & 1u) {
				const uint32_t h0 = tb_hash(k[q]);
				uint32_t h = tb_shash(h0) & (TB_ISLOTS - 1);
				bool found = false;
				for (;;) {
					const unsigned long long cur = s_key[h];
					if (cur == k[q]) { r = s_rank[h]; found = true; break; }
					if (cur == TB_EMPTY) break;
					h = (h + 1) & (TB_ISLOTS - 1);
				}
				if (!found) {
					h = h0 & mask;
					for (uint32_t p = 0;; p++) {
						const ulonglong2 v = __ldg(reinterpret_cast<const ulonglong2 *>(table) + h);
						if (v.x == k[q]) { r = (uint32_t)v.y; break; }
						if (v.x == TB_EMPTY || p == mask) { missing = true; break; }
						h = (h + 1) & mask;
					}
				}
			}
			lo[q >> 1] |= (r & 0xFFFFu) << (16 * (q & 1));
			hi[q >> 2] |= ((r >> 16) & 0xFFu) << (8 * (q & 3));
		}
		const uint64_t o = (uint64_t)c * tpitch + t0;
		*reinterpret_cast<uint4 *>(tl + o) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
		*reinterpret_cast<uint2 *>(th + o) = make_uint2(hi[0], hi[1]);
	}
	if (missing) atomicOr(bad, 1u);
}

namespace {
int tb_grid(int sm_count, uint64_t groups) {
	uint64_t grid = 2ull * (uint64_t)sm_count;                  // two 512-thread CTAs per SM
	{ static const int env_grid = [] { const char *g = getenv("APO_K1_GRID"); return g ? atoi(g) : 0; }(); if (env_grid > 0 && (uint64_t)env_grid < grid) grid = (uint64_t)env_grid; }
	const uint64_t need = (groups + TB_THREADS - 1) / TB_THREADS;
	if (grid > need) grid = need;
	return (int)(grid ? grid : 1);
}
}  // namespace

cudaError_t run_tb_clear(unsigned long long *table, uint64_t slots, cudaStream_t st) {
	uint64_t g = (slots + 255) / 256;
	if (g > 132ull * 32) g = 132ull * 32;
	k_tb_clear<<<(unsigned)g, 256, 0, st>>>(table, slots);
	return cudaGetLastError();
}

cudaError_t run_tb_count(const TbSource &S, unsigned long long *table, uint64_t slots, uint64_t cap, unsigned long long *nkeys,
                         uint32_t *over, int sm_count, cudaStream_t st) {
	const uint64_t groups = (uint64_t)S.C * ((S.T + TB_GROUP - 1) / TB_GROUP);
	if (groups == 0) return cudaSuccess;
	const int smem = (int)(TB_CSLOTS * 12);
	cudaError_t err = allow_big_smem(k_tb_count, smem);
	if (err != cudaSuccess) return err;
	int grid = tb_grid(sm_count, groups);
	const uint64_t min_grid = groups / (1ull << 28) + 1;           // < 2^31 evaluations per CTA: its 32-bit counts cannot wrap
	if ((uint64_t)grid < min_grid) grid = (int)min_grid;
	k_tb_count<<<grid, TB_THREADS, smem, st>>>(S, table, (uint32_t)(slots - 1), cap, nkeys, over);
	return cudaGetLastError();
}

cudaError_t run_tb_compact(const unsigned long long *table, uint64_t slots, unsigned long long *keys, unsigned long long *counts,
                           unsigned long long *n, cudaStream_t st) {
	uint64_t g = (slots + 255) / 256;
	if (g > 132ull * 32) g = 132ull * 32;
	k_tb_compact<<<(unsigned)g, 256, 0, st>>>(table, slots, keys, counts, n);
	return cudaGetLastError();
}

cudaError_t run_tb_insert(const unsigned long long *keys, uint32_t n, unsigned long long *table, uint64_t slots, cudaStream_t st) {
	if (n == 0) return cudaSuccess;
	k_tb_insert<<<(n + 255) / 256, 256, 0, st>>>(keys, n, table, (uint32_t)(slots - 1));
	return cudaGetLastError();
}

cudaError_t run_tb_index(const TbSource &S, const unsigned long long *keys, uint32_t n, const unsigned long long *table, uint64_t slots,
                         unsigned short *tl, unsigned char *th, uint64_t tpitch, uint32_t *bad, int sm_count, cudaStream_t st) {
	const uint64_t groups = (uint64_t)S.C * ((S.T + TB_GROUP - 1) / TB_GROUP);
	if (groups == 0) return cudaSuccess;
	const int smem = (int)(TB_ISLOTS * 12);
	cudaError_t err = allow_big_smem(k_tb_index, smem);
	if (err != cudaSuccess) return err;
	k_tb_index<<<tb_grid(sm_count, groups), TB_THREADS, smem, st>>>(S, keys, n, table, (uint32_t)(slots - 1), tl, th, tpitch, bad);
	return cudaGetLastError();
}

}  // namespace apo
