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
#include "apo_device.cuh"
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
constexpr uint32_t KT_HOT_MAX = 24576;            // 192 KB of shared memory

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

}  // namespace apo
