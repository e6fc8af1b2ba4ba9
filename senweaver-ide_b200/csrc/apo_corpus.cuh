// apo_corpus.cuh — K2 (6-pattern scan + report partials) and K3 (segmented sum + radix top-K) as
// device functions, shared by the stand-alone kernels (k_detect6, k_finalize) and by the scoring
// kernels K1 / K1q, which run the corpus scan on one extra warp per CTA and the finalisation in
// the last CTA to finish (one launch per scoring call).
#pragma once
#include "apo_device.cuh"
#include "apo_kernels.h"

namespace apo {

// Phase stamps of K1h (k_reward9th), in a build with -DAPO_K1H_DIAG only (examples/flagship_launch.py): %globaltimer of every
// CTA at its entry, the end of its pairs (the last stream warp), the end of its digest share, its ticket, and in the
// finalising CTA the start and end of finalize_block and the end of the publish.  Nothing in a product build.
enum { KH_ST_ENTRY, KH_ST_PAIRS, KH_ST_DIGEST, KH_ST_TICKET, KH_ST_FIN0, KH_ST_FIN1, KH_ST_PUBLISH, KH_STAMPS = 8 };
#ifdef APO_K1H_DIAG
constexpr uint32_t KH_STAMP_WORDS = 256 * KH_STAMPS;
static __device__ unsigned long long g_kh_stamp[KH_STAMP_WORDS];
__device__ __forceinline__ unsigned long long kh_now() {
	unsigned long long t;
	asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
	return t;
}
// by thread 0 of the CTA
__device__ __forceinline__ void kh_stamp(int k) {
	if (threadIdx.x == 0 && blockIdx.x < 256) g_kh_stamp[blockIdx.x * KH_STAMPS + k] = kh_now();
}
// by lane 0 of every warp that calls it: the latest
__device__ __forceinline__ void kh_stamp_max(int k) {
	if ((threadIdx.x & 31) == 0 && blockIdx.x < 256) atomicMax(&g_kh_stamp[blockIdx.x * KH_STAMPS + k], kh_now());
}
#else
__device__ __forceinline__ void kh_stamp(int) {}
__device__ __forceinline__ void kh_stamp_max(int) {}
#endif

// First-three-examples slots hold INVERTED record indices (key = ~index, 0 = empty), so that zero-filled memory is
// an armed slot set (one memset arms accumulators, slots and ticket).  Smallest index == largest key.
__device__ __forceinline__ void ex_insert(unsigned long long *slots, unsigned long long key) {
	// keep the 3 largest keys: a key flows down the chain, every slot only increases
	unsigned long long v = key;
#pragma unroll
	for (int k = 0; k < 3; k++) {
		const unsigned long long old = atomicMax(&slots[k], v);
		if (old == 0ull) return;                    // slot was empty: nothing displaced
		v = old < v ? old : v;
	}
}


// Per-thread state of one chunk of <= K2_CHUNK records.  Seven of the nine dimensions are
// categorical (TCS:677-761), so their per-dimension sums (APO:556-565) are kept as packed
// occurrence counters — one 64-bit register per dimension, one small field per category — and
// turned into exact fixed-point sums at flush time: sum = SUM_k count_k * rint(value_k * 2^52),
// an integer product, identical to adding rint(value * 2^52) record by record.
constexpr int K2_CHUNK = 256;      // < 2^9: no packed field (>= 9 bits wide) can overflow inside a chunk

__device__ __forceinline__ void add_i128(long long *dst, __int128 v) {
	const unsigned long long lo = (unsigned long long)v;
	const unsigned long long l0 = lo & 0xffffffffull, l1 = lo >> 32, l2 = (unsigned long long)(long long)(v >> 64);
	if (l0) atomicAdd((unsigned long long *)dst + 0, l0);
	if (l1) atomicAdd((unsigned long long *)dst + 1, l1);
	if (l2) atomicAdd((unsigned long long *)dst + 2, l2);
}
// field f (width bits) of a packed counter, summed over the warp
template <int WIDTH>
__device__ __forceinline__ uint32_t field_sum(unsigned long long pk, int f) {
	return warp_sum_u32((uint32_t)(pk >> (WIDTH * f)) & ((1u << WIDTH) - 1u));
}


// Per-thread accumulators of the corpus scan between two flushes (<= K2_CHUNK records).
struct ScanAcc {
	unsigned long long mTot, mGood, mBad;                    // 5 modes x 12 bits       (APO:519-525)
	unsigned long long c01a, c01b;                            // (fb + 3*err) x 10 bits, endTime unset / set
	unsigned long long c3, c4, c5, c7, c8;                    // 5 slots x 12 bits, slot 4 = not pushed
	unsigned long long c6;                                    // 7 slots x 9 bits, slot 6 = not pushed
	unsigned long long pat;                                   // 6 patterns x 10 bits
	unsigned long long tool[3];
	long long fxR, fxD2;
	uint32_t nValid;
	__device__ __forceinline__ void zero() {
		mTot = mGood = mBad = c01a = c01b = c3 = c4 = c5 = c7 = c8 = c6 = pat = 0ull;
		tool[0] = tool[1] = tool[2] = 0ull; fxR = fxD2 = 0ll; nValid = 0u;
	}
};

// The reward key of a VALID record: its categorical slots and d2 (CatIdx of record_ws_table_t).  Everything the weights touch
// in the corpus report depends on a record through this key alone: the corpus scan (scan_record) takes the weighted sum and
// mask record_ws_table_t computes on the way, the pass over the corpus digest (csrc/apo_kernels.cu k_corpus_digest) recomputes
// them from a stored key (key_ws), and both then run key_reward.
// TCS:777-783 for one key: the weighted sum in push order through the product table (record_ws_table_t's adds, from the
// slots), and the presence mask (the last slot of a group = not pushed).
__device__ __forceinline__ uint32_t key_ws(const CatIdx &ix, double w2, const double *cat, double &ws_out) {
	double ws = cat[CAT_D01 + ix.i01];
	ws = __dadd_rn(ws, __dmul_rn(ix.d2, w2));
	ws = __dadd_rn(ws, cat[CAT_D3 + ix.i3]);
	ws = __dadd_rn(ws, cat[CAT_D4 + ix.i4]);
	ws = __dadd_rn(ws, cat[CAT_D5 + ix.i5]);
	ws = __dadd_rn(ws, cat[CAT_D6 + ix.i6]);
	ws = __dadd_rn(ws, cat[CAT_D7 + ix.i7]);
	ws = __dadd_rn(ws, cat[CAT_D8 + ix.i8]);
	ws_out = ws;
	return 3u | (ix.i3 != 4u ? 0x1cu : 0u) | (ix.i5 != 4u ? 0x20u : 0u) | (ix.i6 != 6u ? 0x40u : 0u) | (ix.i7 != 4u ? 0x80u : 0u) |
	       (ix.i8 != 4u ? 0x100u : 0u);
}
// TCS:784: true when the key's total weight is > 0, with fx = rint(finalReward * 2^52).  ROT: LUT stored at the bank-rotated index.
template <bool ROT>
__device__ __forceinline__ bool key_reward(double ws, uint32_t mask, const double2 *s_lut, long long &fx) {
	const double2 tw = s_lut[ROT ? lut_index(mask) : mask];
	if (!(tw.x > 0.0)) return false;
	fx = to_fx(div_lut<false>(ws, tw));
	return true;
}

// One record of the corpus: tallies, the weighted reward and the per-dimension census, the six 'bad'-gated predicates
// (APO:509-538, 550-565, 644-755).  gi = global index of the record.  ROT: LUT stored at the bank-rotated index.
template <bool ROT>
__device__ __forceinline__ void scan_record(ScanAcc &A, const apo_record &r, unsigned long long gi, unsigned long long *s_ex,
                                            const double *s_cat, const double2 *s_lut, double w2) {
	const bool good = r.feedback == 1, bad = r.feedback == 2;
	const uint32_t msh = 12u * (r.mode < APO_NMODE ? r.mode : 0u);               // APO:627-633
	A.mTot += 1ull << msh; A.mGood += (unsigned long long)good << msh; A.mBad += (unsigned long long)bad << msh;
	A.tool[0] += r.toolCalls; A.tool[1] += r.toolSucc; A.tool[2] += r.toolFail;  // TCS:603-605

	if (r.flags & APO_F_VALID) {                                                 // APO:550, TCS:606
		double ws; CatIdx ix;
		const uint32_t mask = record_ws_table_t<true, true>(r, w2, s_cat, ws, ix);
		long long fx;
		if (key_reward<ROT>(ws, mask, s_lut, fx)) {                              // TCS:784 totalWeight > 0
			A.fxR += fx;
			A.nValid++;
			const unsigned long long one01 = 1ull << (10u * (ix.i01 % 6u));
			if (ix.i01 >= 6u) A.c01b += one01; else A.c01a += one01;
			A.c3 += 1ull << (12u * ix.i3); A.c4 += 1ull << (12u * ix.i4); A.c5 += 1ull << (12u * ix.i5);
			A.c6 += 1ull << (9u * ix.i6); A.c7 += 1ull << (12u * ix.i7); A.c8 += 1ull << (12u * ix.i8);
			A.fxD2 += to_fx(ix.d2);                                              // +0.0 when not pushed
		}
	}
	if (bad) {                                                                   // APO:644-755: every predicate ANDs 'bad'
		const unsigned long long gk = ~gi;                                       // inverted index (see ex_insert)
		const bool hit[APO_NPAT] = {
		    (r.flags & APO_F_ERRORS) != 0,       // P1 APO:644
		    (r.flags & APO_F_FAILSPAN) != 0,     // P2 APO:666-670
		    r.tokens > 10000u,                   // P3 APO:693
		    r.llmCalls > 2u,                     // P4 APO:713
		    r.userMsgs >= 4u,                    // P5 APO:733-734
		    (r.durClass & APO_DC_SLOW) != 0,     // P6 APO:754 (resident records always carry the class)
		};
#pragma unroll
		for (int p = 0; p < APO_NPAT; p++) {
			if (hit[p]) {
				A.pat += 1ull << (10 * p);
				// slice(0,3): first three in corpus order
				if (gk > *((volatile unsigned long long *)&s_ex[3 * p + 2])) ex_insert(&s_ex[3 * p], gk);
			}
		}
	}
}

// The census of counted records -> exact per-dimension sums and counts (APO:556-565): sum = SUM_k count_k * rint(value_k * 2^52)
// per dimension, as adding rint(value * 2^52) record by record.  cnt(g, k) is the count of slot k of group g: g = 0 the
// (feedback, hasErrors, endTime) slot fb + 3 err + 6 ended (TCS:677-691), g = 3..8 the level of dimension g (k = 0..3, d6:
// 0..5); absent slots are never asked for.  nv: the counted records (withReward, the d0 / d1 counts).  Every thread of the
// caller's group calls cnt (it may be a warp collective); `writer` adds into the corpus block corp.  The d2 sum (CORP_DIM + 8)
// and the reward limbs are the caller's.  Shared by the corpus scan (scan_flush) and the digest pass (k_corpus_digest).
template <class Count, class N>
__device__ __forceinline__ void census_flush(Count cnt, N nv, long long *corp, bool writer) {
	// d0 / d1 from the (feedback, hasErrors, endTime) census: TCS:677-691
	__int128 s0 = 0, s1 = 0;
#pragma unroll
	for (int ended = 0; ended < 2; ended++)
#pragma unroll
		for (int err = 0; err < 2; err++)
#pragma unroll
			for (int fb = 0; fb < 3; fb++) {
				const N n = cnt(0, fb + 3 * err + 6 * ended);
				const double d0 = fb == 1 ? 1.0 : (fb == 2 ? -1.0 : 0.0);
				const double d1 = fb == 1 ? 1.0 : (err ? -0.5 : (ended ? 0.8 : 0.5));
				s0 += (__int128)n * to_fx(d0);
				s1 += (__int128)n * to_fx(d1);
			}
	const double lv_rel[4] = {1.0, -0.2, -0.5, -1.0}, lv_cnt[4] = {1.0, 0.3, -0.3, -0.8}, lv_dur[4] = {1.0, 0.5, 0.0, -0.5};
	__int128 s3 = 0, s4 = 0, s5 = 0, s7 = 0, s8 = 0, s6 = 0;
	N n3 = 0, n5 = 0, n6 = 0, n7 = 0, n8 = 0;
#pragma unroll
	for (int k = 0; k < 4; k++) {
		const N a3 = cnt(3, k), a4 = cnt(4, k), a5 = cnt(5, k);
		const N a7 = cnt(7, k), a8 = cnt(8, k);
		s3 += (__int128)a3 * to_fx(lv_rel[k]); s4 += (__int128)a4 * to_fx(lv_cnt[k]); s5 += (__int128)a5 * to_fx(lv_dur[k]);
		s7 += (__int128)a7 * to_fx(lv_dur[k]); s8 += (__int128)a8 * to_fx(lv_cnt[k]);
		n3 += a3; n5 += a5; n7 += a7; n8 += a8;
	}
#pragma unroll
	for (int k = 0; k < 6; k++) {                                                    // TCS:735: max(-1, 1 - k*0.4)
		const N a6 = cnt(6, k);
		double ef = __dadd_rn(1.0, -__dmul_rn((double)k, 0.4));
		ef = ef < -1.0 ? -1.0 : ef;
		s6 += (__int128)a6 * to_fx(ef);
		n6 += a6;
	}
	if (writer) {
		const __int128 sums[APO_NDIM] = {s0, s1, 0, s3, s4, s5, s6, s7, s8};
		const N cnts[APO_NDIM] = {nv, nv, n3, n3, n3, n5, n6, n7, n8};                   // d2,d3,d4 are pushed together (TCS:695)
#pragma unroll
		for (int i = 0; i < APO_NDIM; i++) {
			if (i != 2) add_i128(corp + CORP_DIM + 4 * i, sums[i]);
			if (cnts[i]) atomicAdd((unsigned long long *)corp + CORP_DIM + 4 * i + 3, (unsigned long long)cnts[i]);
		}
		if (nv) atomicAdd((unsigned long long *)corp + CORP_REWARD + 3, (unsigned long long)nv);
	}
}

// Flush one chunk: warp-reduce every field, lane 0 turns counts into exact sums.  Full-warp collective.
__device__ __forceinline__ void scan_flush(const ScanAcc &A, long long *corp, int lane) {
	uint32_t good = 0, badn = 0, total = 0;
#pragma unroll
	for (int m = 0; m < APO_NMODE; m++) {
		const uint32_t a = field_sum<12>(A.mTot, m), g = field_sum<12>(A.mGood, m), b = field_sum<12>(A.mBad, m);
		if (lane == 0) {
			if (a) atomicAdd((unsigned long long *)corp + CORP_MODE + 3 * m, (unsigned long long)a);
			if (g) atomicAdd((unsigned long long *)corp + CORP_MODE + 3 * m + 1, (unsigned long long)g);
			if (b) atomicAdd((unsigned long long *)corp + CORP_MODE + 3 * m + 2, (unsigned long long)b);
		}
		total += a; good += g; badn += b;
	}
	if (lane == 0) {                                                                 // APO:513-516
		if (good) atomicAdd((unsigned long long *)corp + CORP_TALLY, (unsigned long long)good);
		if (badn) atomicAdd((unsigned long long *)corp + CORP_TALLY + 1, (unsigned long long)badn);
		if (total - good - badn) atomicAdd((unsigned long long *)corp + CORP_TALLY + 2, (unsigned long long)(total - good - badn));
	}
#pragma unroll
	for (int p = 0; p < APO_NPAT; p++) {
		const uint32_t n = field_sum<10>(A.pat, p);
		if (lane == 0 && n) atomicAdd((unsigned long long *)corp + CORP_PAT + p, (unsigned long long)n);
	}
#pragma unroll
	for (int i = 0; i < 3; i++) {
		const unsigned long long s = warp_sum_u64(A.tool[i]);
		if (lane == 0 && s) atomicAdd((unsigned long long *)corp + CORP_TOOL + i, s);
	}
	{   // finalReward sum and count (APO:550-553)
		Acc128 a; a.lo = (unsigned long long)A.fxR; a.hi = A.fxR >> 63;
		flush_acc128(a, corp + CORP_REWARD, lane);
		Acc128 b; b.lo = (unsigned long long)A.fxD2; b.hi = A.fxD2 >> 63;
		flush_acc128(b, corp + CORP_DIM + 4 * 2, lane);
	}
	const uint32_t nv = warp_sum_u32(A.nValid);
	census_flush(
	    [&](int g, int k) -> uint32_t {
		    switch (g) {
		    case 0: return field_sum<10>(k >= 6 ? A.c01b : A.c01a, k % 6);
		    case 3: return field_sum<12>(A.c3, k);
		    case 4: return field_sum<12>(A.c4, k);
		    case 5: return field_sum<12>(A.c5, k);
		    case 6: return field_sum<9>(A.c6, k);
		    case 7: return field_sum<12>(A.c7, k);
		    default: return field_sum<12>(A.c8, k);
		    }
	    },
	    nv, corp, lane == 0);
}

// One warp's share of the corpus: records t = first + lane, first + lane + stride, ...  All 32 lanes stay
// in the loop together (full-warp collectives in the flush).  s_ex: 18 shared-memory slots (first three
// matches of each pattern as inverted indices, 0 = empty) shared by the caller's warps; s_cat / s_lut: the categorical
// product table and the {total weight, reciprocal} LUT (ROT: LUT stored at the bank-rotated index).
template <bool ROT>
__device__ __forceinline__ void corpus_scan_warp(const K2Params &P, uint64_t first, uint64_t stride, unsigned long long *s_ex,
                                                 const double *s_cat, const double2 *s_lut, int lane) {
	const double w2 = P.W.w[2];
	long long *corp = P.acc + (uint64_t)ACC_PER_CAND * P.C;
	const uint4 *src = reinterpret_cast<const uint4 *>(P.recs);
	uint64_t t = first + lane;
	const uint64_t per_lane = first < P.T ? (P.T - first + stride - 1) / stride : 0;   // iterations of lane 0 (the most any lane runs)
	const uint64_t rounds = (per_lane + K2_CHUNK - 1) / K2_CHUNK;

	for (uint64_t round = 0; round < rounds; round++) {
		ScanAcc A; A.zero();
		// software pipeline: the next record of this thread is in flight while the current one is scored
		union Rec { uint4 q[2]; apo_record r; } nxt;
		if (t < P.T) { nxt.q[0] = __ldg(src + 2 * t); nxt.q[1] = __ldg(src + 2 * t + 1); }
		for (int it = 0; it < K2_CHUNK && t < P.T; it++, t += stride) {
			Rec u = nxt;
			if (it + 1 < K2_CHUNK && t + stride < P.T) { nxt.q[0] = __ldg(src + 2 * (t + stride)); nxt.q[1] = __ldg(src + 2 * (t + stride) + 1); }
			scan_record<ROT>(A, u.r, P.idx_base + t, s_ex, s_cat, s_lut, w2);
		}
		scan_flush(A, corp, lane);
	}
}

// After every scanning warp of the CTA has flushed: push the CTA's first-three examples to the global
// scratch, take a ticket, and let the last CTA publish this rank's examples and finalise (segmented sum +
// top-K; at > 1 rank after the peer-memory join of the partial vectors).
// Must be called by every thread of the CTA (it synchronises the block).
static __device__ void finalize_and_publish(const FinalizeParams &F, unsigned long long *s_scratch, uint32_t scratch_keys);

// s_scratch / scratch_keys: shared memory the caller no longer needs at this point (a free stage buffer, the LUT of the
// grid-stride kernel), lent to the finalisation for its small-C top-K.
__device__ __forceinline__ void corpus_tail(const K2Params &P, const unsigned long long *s_ex, bool *s_last,
                                            unsigned long long *s_scratch = nullptr, uint32_t scratch_keys = 0) {
	// Fences: one thread fences AFTER a block barrier instead of every thread fencing before it — the barrier makes the
	// block's earlier writes (the warps' atomics) visible to that thread and the fence is cumulative, which is the pattern
	// of a grid-wide barrier; 704 MEMBARs per CTA were most of a small call's device time.
	const int tid = threadIdx.x;
	long long *corp = P.acc + (uint64_t)ACC_PER_CAND * P.C;
	__syncthreads();
	if (tid < APO_NPAT) {
#pragma unroll
		for (int k = 0; k < 3; k++) {
			const unsigned long long v = s_ex[3 * tid + k];
			if (v != 0ull && v > P.ex_scratch[3 * tid + 2]) ex_insert(&P.ex_scratch[3 * tid], v);
		}
	}
	__syncthreads();
	if (tid == 0) {
		__threadfence();
		const unsigned int ticket = atomicAdd(P.ticket, 1u);
		*s_last = (ticket == gridDim.x - 1);
		if (*s_last) __threadfence();                             // acquire side: the other CTAs' flushes are visible from here on
		kh_stamp(KH_ST_TICKET);
	}
	__syncthreads();
	if (!*s_last) return;
	if (tid < APO_NPAT * 3) {
		const unsigned long long v = *((volatile unsigned long long *)&P.ex_scratch[tid]);
		corp[CORP_EX + 18 * P.rank + tid] = v == 0ull ? 0ll : (long long)(~v + 1);     // index + 1, 0 = none
	}
	if (tid == 0) { corp[CORP_NREC] = (long long)P.T; *P.ticket = 0; }
	__syncthreads();                                              // block-scope visibility is all the finalising CTA needs (it reads through L2)
	if (P.fuse_finalize) finalize_and_publish(P.fin, s_scratch, scratch_keys);
}

// ---------------------------------------------------------------- the corpus digest pass (apo_kernels.h CorpusDigestParams)
__device__ __forceinline__ CatIdx cd_key(const ulonglong2 &e) {
	CatIdx ix;
	const uint32_t s = (uint32_t)e.y;
	ix.i01 = s & 15u; ix.i3 = (s >> 4) & 7u; ix.i4 = (s >> 7) & 7u; ix.i5 = (s >> 10) & 7u;
	ix.i6 = (s >> 13) & 7u; ix.i7 = (s >> 16) & 7u; ix.i8 = (s >> 19) & 7u;
	ix.d2 = __longlong_as_double((long long)e.x);
	return ix;
}

// census counters of the digest pass: group g slot k (the slots census_flush asks for)
__device__ __forceinline__ int cd_census(int g, int k) { return g == 0 ? k : g == 6 ? 24 + k : g < 6 ? 12 + 4 * (g - 3) + k : 30 + 4 * (g - 7) + k; }
constexpr int CD_CENSUS = 38;
// c into the 64-bit counter {lo, hi} of shared memory with native 32-bit adds (a 64-bit shared-memory add is a CAS loop, and
// every entry of a CTA meets the same few counters): the low word's carry goes to the high word
__device__ __forceinline__ void cd_add(uint32_t *lo, uint32_t *hi, unsigned long long c) {
	const uint32_t l = (uint32_t)c, h = (uint32_t)(c >> 32);
	const uint32_t carry = atomicAdd(lo, l) > 0xFFFFFFFFu - l ? 1u : 0u;
	if (h + carry) atomicAdd(hi, h + carry);
}

// the block's census counters -> exact dimension sums (census_flush), by one thread; a call of its own keeps its 128-bit sums
// out of the register budget of the kernels that run the pass (K1h: 64 registers)
static __device__ __noinline__ void cd_census_flush(const uint32_t *s_lo, const uint32_t *s_hi, long long *corp) {
	auto count = [&](int j) { return (unsigned long long)s_hi[j] << 32 | s_lo[j]; };
	census_flush([&](int g, int k) { return count(cd_census(g, k)); }, count(CD_CENSUS), corp, true);
}

// One call's corpus words from the digest: each CTA takes a contiguous share of the entries and runs, per entry, what
// scan_record runs per record (key_ws, key_reward), times the entry's count; CTA 0 adds the fixed words and seeds its example
// slots; then the tail of the stand-alone scan (ticket, examples, the last CTA finalises when the call asks for it).  Run by
// the stand-alone k_corpus_digest on every warp of its CTAs (corpus_digest_block) and by K1h (k_reward9th) on one warp of
// every CTA while the other warps stream the pairs (cd_warp, then cd_tail).  P.fixed == NULL: no corpus words (a call
// without a corpus report), only the tail.
struct CdShared {
	unsigned long long ex[APO_NPAT * 3];
	double cat[CAT_WORDS];
	double2 lut[512];
	uint32_t lo[CD_CENSUS + 1], hi[CD_CENSUS + 1];   // + the counted records
	unsigned long long part[32][6];                  // per warp that ran entries: the limb sums of the reward and of d2
	bool last;
};
// one instance per CTA, shared by the parts below
__device__ __forceinline__ CdShared &cd_shared() {
	__shared__ CdShared s;
	return s;
}

// the CTA's examples, census counters and tables, by threads t = 0 .. nt - 1 of the caller's group (the caller syncs the group)
__device__ __forceinline__ void cd_setup(const CorpusDigestParams &P, CdShared &S, int t, int nt) {
	const K2Params &K = P.k2;
	long long *corp = K.acc + (uint64_t)ACC_PER_CAND * K.C;
	for (int i = t; i < APO_NPAT * 3; i += nt) S.ex[i] = blockIdx.x == 0 && P.fixed ? (unsigned long long)P.fixed[CD_FIXED + i] : 0ull;
	for (int i = t; i <= CD_CENSUS; i += nt) { S.lo[i] = 0u; S.hi[i] = 0u; }
	for (int i = t; i < CAT_WORDS; i += nt) S.cat[i] = K.lut[1024 + i];
	for (int i = t; i < 512; i += nt) S.lut[i] = make_double2(K.lut[i], K.lut[512 + i]);
	if (blockIdx.x == 0 && P.fixed)
		for (int i = t; i < CD_FIXED; i += nt)
			if (P.fixed[i]) atomicAdd((unsigned long long *)corp + CORP_TALLY + i, (unsigned long long)P.fixed[i]);
}

constexpr int CD_UNROLL = 4;   // entries in flight per lane

// One warp's entries i = first + lane, first + lane + stride, ... below hi into the census counters; its limb sums go to
// S.part[row].  Full-warp collective.
static __device__ __noinline__ void cd_entries(const CorpusDigestParams &P, CdShared &S, uint64_t first, uint64_t stride, uint64_t hi,
                                               int row) {
	const int lane = threadIdx.x & 31;
	const double w2 = P.k2.W.w[2];
	Acc128 R, D2; R.zero(); D2.zero();
	for (uint64_t i0 = first + lane; i0 < hi; i0 += CD_UNROLL * stride) {
		ulonglong2 e[CD_UNROLL];
#pragma unroll
		for (int u = 0; u < CD_UNROLL; u++) {
			const uint64_t i = i0 + u * stride;
			e[u] = i < hi ? P.ent[i] : make_ulonglong2(0ull, 0ull);
		}
#pragma unroll 1
		for (int u = 0; u < CD_UNROLL; u++) {
			if (i0 + u * stride >= hi) break;
			const CatIdx ix = cd_key(e[u]);
			const unsigned long long c = e[u].y >> CD_COUNT_SHIFT;
			double ws;
			const uint32_t mask = key_ws(ix, w2, S.cat, ws);
			long long fx;
			if (key_reward<false>(ws, mask, S.lut, fx)) {             // TCS:784 totalWeight > 0
				acc_add_mul(R, c, fx);
				acc_add_mul(D2, c, to_fx(ix.d2));                     // +0.0 when not pushed
				auto add = [&](int j) { cd_add(&S.lo[j], &S.hi[j], c); };
				add(CD_CENSUS);
				add(cd_census(0, (int)ix.i01));
				if (ix.i3 < 4u) { add(cd_census(3, (int)ix.i3)); add(cd_census(4, (int)ix.i4)); }
				if (ix.i5 < 4u) add(cd_census(5, (int)ix.i5));
				if (ix.i6 < 6u) add(cd_census(6, (int)ix.i6));
				if (ix.i7 < 4u) add(cd_census(7, (int)ix.i7));
				if (ix.i8 < 4u) add(cd_census(8, (int)ix.i8));
			}
		}
	}
	const unsigned long long v[6] = {warp_sum_u64(R.lo & 0xffffffffull), warp_sum_u64(R.lo >> 32), warp_sum_u64((unsigned long long)R.hi),
	                                 warp_sum_u64(D2.lo & 0xffffffffull), warp_sum_u64(D2.lo >> 32), warp_sum_u64((unsigned long long)D2.hi)};
	if (lane == 0)
		for (int k = 0; k < 6; k++) S.part[row][k] = v[k];
}

// After every warp that ran entries has written its row of S.part (rows [0, nrows)) and its census adds, and the caller has
// synced them: `who` 0 turns the census into dimension sums, 1..6 add one limb each, summed over the rows (the limbs are summed
// over the CTA first: one global atomic per limb and CTA, thousands of warps adding into the same six words serialise in L2;
// the high limb wraps as a signed sum, as flush_acc128 adds it).
__device__ __forceinline__ void cd_flush(const CorpusDigestParams &P, const CdShared &S, int nrows, int who) {
	long long *corp = P.k2.acc + (uint64_t)ACC_PER_CAND * P.k2.C;
	if (who == 0) cd_census_flush(S.lo, S.hi, corp);
	else if (who >= 1 && who <= 6) {
		const int k = who - 1;
		unsigned long long sum = 0;
		for (int w = 0; w < nrows; w++) sum += S.part[w][k];
		if (sum) atomicAdd((unsigned long long *)corp + (k < 3 ? CORP_REWARD + k : CORP_DIM + 4 * 2 + k - 3), sum);
	}
}

// The tail after the pass: ticket, examples, the last CTA finalises.  Block-wide; its first barrier orders the pass's adds
// before the ticket.
__device__ __forceinline__ void cd_tail(const CorpusDigestParams &P, CdShared &S) {
	corpus_tail(P.k2, S.ex, &S.last, reinterpret_cast<unsigned long long *>(S.lut), 1024u);   // the LUT (8 KB) is done with: scratch of the tail
}

// The whole pass on one warp of the CTA (K1h): set-up, this CTA's share of the entries, the flush.  The caller then runs cd_tail
// on every thread of the CTA.
static __device__ __noinline__ void cd_warp(const CorpusDigestParams &P) {
	CdShared &S = cd_shared();
	const int lane = threadIdx.x & 31;
	cd_setup(P, S, lane, 32);
	__syncwarp();
	const uint64_t n = P.fixed ? *P.n : 0, lo = n * blockIdx.x / gridDim.x, hi = n * (blockIdx.x + 1ull) / gridDim.x;
	cd_entries(P, S, lo, 32, hi, 0);
	__syncwarp();
	cd_flush(P, S, 1, lane);
}

// The pass on every warp of the CTA (the stand-alone k_corpus_digest), then the tail.  Block-wide; every thread of every CTA
// of the launch must enter.  Works for any blockDim.x that is a multiple of 32 (<= 1024).
static __device__ __noinline__ void corpus_digest_block(const CorpusDigestParams &P) {
	CdShared &S = cd_shared();
	const int tid = threadIdx.x;
	cd_setup(P, S, tid, blockDim.x);
	__syncthreads();
	const uint64_t n = P.fixed ? *P.n : 0, lo = n * blockIdx.x / gridDim.x, hi = n * (blockIdx.x + 1ull) / gridDim.x;
	cd_entries(P, S, lo + (tid & ~31), blockDim.x, hi, tid >> 5);
	__syncthreads();
	cd_flush(P, S, blockDim.x >> 5, tid == 0 ? 0 : tid >= 32 && tid < 38 ? tid - 31 : -1);
	cd_tail(P, S);
}

__device__ __forceinline__ unsigned long long score_key(double s) {
	const unsigned long long b = (unsigned long long)__double_as_longlong(s);
	return (b >> 63) ? ~b : (b | 0x8000000000000000ull);     // ascending order-preserving map
}

// The numeric rules of a report, shared by the corpus report (build_report) and the per-candidate breakdown
// (csrc/apo_cand.cu k_cand_report) so that the two cannot drift apart.
// good / (good + bad), 0 when both are 0 (APO:546-547, APO:541-544)
__device__ __forceinline__ double report_good_rate(uint64_t good, uint64_t bad) {
	const uint64_t twf = good + bad;
	return twf > 0 ? __ddiv_rn((double)good, (double)twf) : 0.0;
}
// rewardSum / withReward, NaN (null) when nothing carried a reward (APO:550-553)
__device__ __forceinline__ double report_avg_reward(double rsum, uint64_t nrew) {
	return nrew > 0 ? __ddiv_rn(rsum, (double)nrew) : __longlong_as_double(0x7ff8000000000000ll);
}
// rewardByDimension entry from its exact (l0, l1, l2, count) words: APO:556-568 + rules APO:575,591,802,819
__device__ __forceinline__ apo_dimstat report_dimstat(const long long l[4]) {
	apo_dimstat D;
	D.sum = limbs_to_double(l);
	D.count = (uint64_t)l[3];
	D.avg = D.count > 0 ? __ddiv_rn(D.sum, (double)D.count) : 0.0;                       // APO:567
	D.low_flag = (D.count >= 5 && D.avg < -0.3) ? 1 : 0;                                 // APO:575
	D.low_severity = D.avg < -0.5 ? 2 : 1;                                               // APO:591
	D.sugg_flag = (D.count >= 3 && D.avg < 0.0) ? 1 : 0;                                 // APO:802
	D.sugg_priority = D.avg < -0.5 ? 2 : 1;                                              // APO:819
	for (int k = 0; k < 4; k++) D.pad[k] = 0;
	return D;
}

// APO:498-625 / TCS:596-626 from the joined corpus block.  Block-wide: the block's words below CORP_EX are staged into s_corp
// (shared memory the caller lends, CORP_EX words) with one coalesced pass (a single thread loading them one by one between its
// stores to the report pays a round trip to L2 per word), then thread 0 the tallies, threads 1..9 one dimension each, threads
// 10..15 one pattern each.
static __device__ void build_report(const FinalizeParams &F, const long long *corp_g, long long *s_corp) {
	const long long *corp = s_corp;
	apo_corpus_report &R = *F.report;
	const int tid = threadIdx.x;
	for (int i = tid; i < CORP_EX; i += blockDim.x) s_corp[i] = __ldcg(corp_g + i);
	__syncthreads();
	if (tid == 0) {
		R.total = (uint64_t)corp[CORP_NREC];
		const uint64_t good = (uint64_t)corp[CORP_TALLY], bad = (uint64_t)corp[CORP_TALLY + 1];
		R.good = good; R.bad = bad; R.none = (uint64_t)corp[CORP_TALLY + 2];
		R.goodRate = report_good_rate(good, bad);                                                // APO:546-547
		for (int m = 0; m < APO_NMODE; m++) {
			uint64_t v[3];
			for (int k = 0; k < 3; k++) { v[k] = (uint64_t)corp[CORP_MODE + 3 * m + k]; R.byMode[m][k] = v[k]; }
			R.byModeGoodRate[m] = report_good_rate(v[1], v[2]);                                  // APO:541-544
		}
		long long l[4];
		for (int q = 0; q < 4; q++) l[q] = corp[CORP_REWARD + q];
		const uint64_t nrew = (uint64_t)l[3];
		const double rsum = limbs_to_double(l);
		R.withReward = nrew; R.rewardSum = rsum;
		R.avgReward = report_avg_reward(rsum, nrew);
		const uint64_t tc = (uint64_t)corp[CORP_TOOL], ts = (uint64_t)corp[CORP_TOOL + 1];
		R.toolCalls = tc; R.toolSucc = ts; R.toolFail = (uint64_t)corp[CORP_TOOL + 2];
		R.toolSuccessRate = tc > 0 ? __ddiv_rn((double)ts, (double)tc)                          // TCS:624
		                           : __longlong_as_double(0x7ff8000000000000ll);
	} else if (tid <= APO_NDIM) {
		const int i = tid - 1;
		long long l[4];
		for (int q = 0; q < 4; q++) l[q] = corp[CORP_DIM + 4 * i + q];
		R.dim[i] = report_dimstat(l);
	} else if (tid <= APO_NDIM + APO_NPAT) {
		const int p = tid - 1 - APO_NDIM;
		const uint64_t minc[APO_NPAT] = {2, 2, 3, 2, 2, 2};                                      // APO:645,671,695,715,736,756
		const uint64_t bad = (uint64_t)corp[CORP_TALLY + 1];
		apo_pattern Q;
		Q.count = bad == 0 ? 0 : (uint64_t)corp[CORP_PAT + p];                                  // APO:641
		Q.flag = Q.count >= minc[p] ? 1 : 0;
		uint8_t sev = 1;
		if (p == 0 || p == 1) sev = Q.count >= 5 ? 2 : 1;                                    // APO:650,676
		else if (p == 3) sev = 2;                                                            // APO:720
		else if (p == 4) sev = Q.count >= 4 ? 2 : 1;                                         // APO:741
		Q.severity = sev;
		for (int k = 0; k < 6; k++) Q.pad[k] = 0;
		// first three in corpus order: ranks hold disjoint ascending index ranges
		int got = 0;
		for (int k = 0; k < 3; k++) Q.examples[k] = -1;
		for (int r = 0; r < F.nranks && got < 3; r++) {
			long long v[3];
			for (int k = 0; k < 3; k++) v[k] = __ldcg(corp_g + CORP_EX + 18 * r + 3 * p + k);
			for (int k = 0; k < 3 && got < 3; k++) if (v[k] > 0) Q.examples[got++] = v[k] - 1;
		}
		R.pat[p] = Q;
	}
}

// Block-wide; every thread of the calling block must enter.  Works for any blockDim.x
// that is a multiple of 32 (<= 1024).
static __device__ __noinline__ void finalize_block(const FinalizeParams &F, unsigned long long *s_scratch, uint32_t scratch_keys) {
	__shared__ __align__(8) unsigned int s_hist[256];          // also the report's stage (build_report), before the top-K
	__shared__ unsigned long long s_prefix;
	__shared__ unsigned int s_need, s_base_gt, s_base_eq, s_warp_gt[32], s_warp_eq[32];
	const int tid = threadIdx.x, nth = blockDim.x, lane = tid & 31, warp = tid >> 5, nwarp = nth >> 5;
	const uint32_t C = F.C;
	const long long *acc = F.acc;

	// 1. segmented sum: limbs -> score[c] = sum / count  (APO:550-553 per candidate)
	for (uint32_t c = tid; c < C; c += nth) {
		long long l[4];
#pragma unroll
		for (int q = 0; q < 4; q++) l[q] = __ldcg(acc + (uint64_t)ACC_PER_CAND * c + q);
		const uint64_t n = (uint64_t)l[3];
		const double s = n > 0 ? __ddiv_rn(limbs_to_double(l), (double)n) : __longlong_as_double(0xfff0000000000000ll);
		F.scores[c] = s;
		F.counts[c] = n;
		F.keys[c] = score_key(s);
		if (C <= scratch_keys) s_scratch[c] = score_key(s);
	}
	static_assert(CORP_EX * sizeof(long long) <= sizeof(s_hist), "the report's stage fits the histogram");
	if (F.with_corpus) build_report(F, acc + (uint64_t)ACC_PER_CAND * C, reinterpret_cast<long long *>(s_hist));
	__syncthreads();
	const uint32_t K = F.K < C ? F.K : C;
	if (K == 0) return;

	// Small beams (the reference's are 4 wide, APO:288): rank every candidate by counting over the keys held in shared memory —
	// position = #{better score, or equal score and lower index} — and let the first K write themselves out.  One barrier
	// instead of the eight histogram passes of the radix select below (12 us of a 4 x 1000 call).
	if (C <= scratch_keys) {
		for (uint32_t i = tid; i < C; i += nth) {
			const unsigned long long ki = s_scratch[i];
			uint32_t rank = 0;
			for (uint32_t j = 0; j < C; j++) {
				const unsigned long long kj = s_scratch[j];
				rank += (kj > ki || (kj == ki && j < i)) ? 1u : 0u;
			}
			if (rank < K) F.topk[rank] = (int32_t)i;
		}
		return;
	}

	// 2. radix select (8-bit digits, MSB first): key of the K-th best candidate
	if (tid == 0) { s_prefix = 0; s_need = K; }
	__syncthreads();
	for (int pass = 0; pass < 8; pass++) {
		const int shift = 56 - 8 * pass;
		for (int i = tid; i < 256; i += nth) s_hist[i] = 0;
		__syncthreads();
		const unsigned long long prefix = s_prefix;
		const unsigned long long maskhi = pass == 0 ? 0ull : (~0ull << (shift + 8));
		for (uint32_t c = tid; c < C; c += nth) {
			const unsigned long long k = F.keys[c];
			if ((k & maskhi) == prefix) atomicAdd(&s_hist[(k >> shift) & 255], 1u);
		}
		__syncthreads();
		if (warp == 0) {
			// the digit d whose suffix count first reaches `need`, scanning 255 -> 0: lane l owns bins [8l, 8l+8)
			unsigned int h[8], tot = 0;
#pragma unroll
			for (int j = 0; j < 8; j++) { h[j] = s_hist[8 * lane + j]; tot += h[j]; }
			unsigned int suf = tot;                                   // sum over lanes >= this one
#pragma unroll
			for (int o = 1; o < 32; o <<= 1) {
				const unsigned int v = __shfl_down_sync(0xffffffffu, suf, o);
				if (lane + o < 32) suf += v;
			}
			const unsigned int need = s_need, above = suf - tot;
			const bool here = above < need && need <= suf;
			const unsigned int any = __ballot_sync(0xffffffffu, here);
			__syncwarp();                                             // every lane has read s_need before one of them rewrites it
			if (here || (any == 0u && lane == 0)) {                   // (any == 0 cannot happen: need <= #keys under the prefix)
				unsigned int rem = need - (here ? above : 0u);
				int j = 7;
				for (; j > 0; j--) {
					if (h[j] >= rem) break;
					rem -= h[j];
				}
				s_need = rem;
				s_prefix = prefix | ((unsigned long long)(8 * lane + j) << shift);
			}
		}
		__syncthreads();
	}
	const unsigned long long kth = s_prefix;       // K-th largest key
	const unsigned int need_eq = s_need;           // how many candidates equal to it are taken (lowest indices)

	// 3. ordered compaction: all keys > kth, plus the first need_eq keys == kth, by index
	if (tid == 0) { s_base_gt = 0; s_base_eq = 0; }
	__syncthreads();
	const unsigned int n_gt = K - need_eq;
	for (uint32_t c0 = 0; c0 < C; c0 += nth) {
		const uint32_t c = c0 + tid;
		const unsigned long long k = c < C ? F.keys[c] : 0ull;
		const bool gt = c < C && k > kth, eq = c < C && k == kth;
		const unsigned int bgt = __ballot_sync(0xffffffffu, gt), beq = __ballot_sync(0xffffffffu, eq);
		if (lane == 0) { s_warp_gt[warp] = __popc(bgt); s_warp_eq[warp] = __popc(beq); }
		__syncthreads();
		unsigned int ogt = s_base_gt, oeq = s_base_eq;
		for (int w = 0; w < warp; w++) { ogt += s_warp_gt[w]; oeq += s_warp_eq[w]; }
		const unsigned int lt = (1u << lane) - 1u;
		const unsigned int pgt = ogt + __popc(bgt & lt), peq = oeq + __popc(beq & lt);
		if (gt) { F.sel_key[pgt] = k; F.sel_idx[pgt] = (int32_t)c; }
		if (eq && peq < need_eq) { F.sel_key[n_gt + peq] = k; F.sel_idx[n_gt + peq] = (int32_t)c; }
		__syncthreads();
		if (tid == 0) {
			unsigned int a = 0, b = 0;
			for (int w = 0; w < nwarp; w++) { a += s_warp_gt[w]; b += s_warp_eq[w]; }
			s_base_gt += a; s_base_eq += b;
		}
		__syncthreads();
	}

	// 4. order the K winners: score descending, ties -> lower index (rank by counting)
	for (uint32_t i = tid; i < K; i += nth) {
		const unsigned long long ki = F.sel_key[i];
		const int32_t ci = F.sel_idx[i];
		uint32_t rank = 0;
		for (uint32_t j = 0; j < K; j++) {
			const unsigned long long kj = F.sel_key[j];
			rank += (kj > ki || (kj == ki && F.sel_idx[j] < ci)) ? 1u : 0u;
		}
		F.topk[rank] = ci;
	}
}

// ---------------------------------------------------------------- cross-rank join over peer memory
__device__ __forceinline__ unsigned long long globaltimer_ns() {
	unsigned long long t;
	asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
	return t;
}
__device__ __forceinline__ void st_release_sys(unsigned long long *p, unsigned long long v) {
	asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long *p) {
	unsigned long long v;
	asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
	return v;
}
__device__ __forceinline__ long long ld_relaxed_sys(const long long *p) {
	long long v;
	asm volatile("ld.relaxed.sys.global.s64 %0, [%1];" : "=l"(v) : "l"(p));      // no memory clobber: independent loads may be in flight together
	return v;
}

constexpr unsigned long long PEER_TIMEOUT_NS = 20ull * 1000 * 1000 * 1000;   // a rank that never arrives: report, do not hang

// Block-wide.  Returns false when a peer did not arrive within PEER_TIMEOUT_NS.
static __device__ bool peer_join(const JoinParams &J, const long long *acc_local, ResultMeta *meta) {
	__shared__ int s_ok;
	const int tid = threadIdx.x, nth = blockDim.x;
	long long *mine = J.slot[J.rank];
	if (tid == 0) s_ok = 1;
	const unsigned long long t0 = globaltimer_ns();
	// 1. publish this rank's partials (they were produced by other CTAs' atomics: read them from L2)
	for (uint32_t i = tid; i < J.words / 2; i += nth)               // the vector has an even number of words and 16-byte aligned slots
		reinterpret_cast<longlong2 *>(mine)[i] = __ldcg(reinterpret_cast<const longlong2 *>(acc_local) + i);
	__syncthreads();
	// 2. raise this rank's flag in every rank's block (remote stores), 3. wait for every rank's flag in ours (local loads).
	//    The signalling threads release at system scope after the barrier (cumulative over the block's slot writes).
	if (tid < J.nranks) {
		st_release_sys(J.flag[tid] + J.rank, J.epoch);            // release at system scope: fence + store (SASS: MEMBAR.ALL.SYS; STG.STRONG.SYS)
		const unsigned long long *f = J.flag[J.rank] + tid;
		while (ld_acquire_sys(f) < J.epoch) {
			if (globaltimer_ns() - t0 > PEER_TIMEOUT_NS) { s_ok = 0; break; }
			__nanosleep(64);
		}
	}
	// while those threads wait (tens of microseconds of launch skew between the ranks), a second warp touches every peer's slot:
	// the first access to a peer mapping pays a page-table walk over NVLink (~2.5 us each, serial in the reduce below otherwise)
	if (tid >= 32 && tid < 32 + J.nranks) {
		long long sink = ld_relaxed_sys(J.slot[tid - 32]);
		asm volatile("" ::"l"(sink));
	}
	__syncthreads();
	const unsigned long long t1 = globaltimer_ns();
	if (!s_ok) { if (tid == 0) { meta->status = 1u; meta->join_wait_us = (float)((t1 - t0) * 1e-3); meta->join_reduce_us = 0.f; } return false; }
	// 4. sum the slots of all ranks (NVLink peer loads; integers: any order gives the same bits)
	//    16-byte L2 loads (ld.global.cg: no L1, served by the owning GPU's L2 — coherent, and ordered after the acquire above by the
	//    barrier), a warp reads 512 contiguous bytes per peer, and all eight peers' loads of a pair are in flight before the first add.
	//    (8-byte ld.relaxed.sys loads are issued request by request.)
	for (uint32_t i = tid; i < J.words / 2; i += nth) {
		longlong2 v[PEER_MAX];
#pragma unroll
		for (int r = 0; r < PEER_MAX; r++) v[r] = r < J.nranks ? __ldcg(reinterpret_cast<const longlong2 *>(J.slot[r]) + i) : make_longlong2(0, 0);
		longlong2 sum = make_longlong2(0, 0);
#pragma unroll
		for (int r = 0; r < PEER_MAX; r++) { sum.x += v[r].x; sum.y += v[r].y; }
		reinterpret_cast<longlong2 *>(J.joined)[i] = sum;
	}
	__syncthreads();
	// tell every peer that this rank no longer reads its slot (only consulted when a peer tears its block down)
	// (a relaxed store: the loads above have returned their values — they fed the stores to `joined` before the barrier)
	if (tid < J.nranks) asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(J.flag[tid] + PEER_MAX + J.rank), "l"(J.epoch) : "memory");
	if (tid == 0) { meta->status = 0u; meta->join_wait_us = (float)((t1 - t0) * 1e-3); meta->join_reduce_us = (float)((globaltimer_ns() - t1) * 1e-3); }
	return true;
}

// join (> 1 rank) -> segmented sum + report + top-K -> result block written to the caller's page-locked buffer.
static __device__ void finalize_and_publish(const FinalizeParams &F0, unsigned long long *s_scratch, uint32_t scratch_keys) {
	FinalizeParams F = F0;
	ResultMeta *meta = reinterpret_cast<ResultMeta *>(F.result_base + F.meta_off);
	bool ok = true;
	if (F.join.nranks > 1) {
		ok = peer_join(F.join, F.acc, meta);
		F.acc = F.join.joined;
	} else if (threadIdx.x == 0) { meta->status = 0u; meta->pad = 0u; meta->join_wait_us = 0.f; meta->join_reduce_us = 0.f; }
	const unsigned long long tf0 = globaltimer_ns();
	kh_stamp(KH_ST_FIN0);
	if (ok) finalize_block(F, s_scratch, scratch_keys);
	__syncthreads();
	const unsigned long long tf1 = globaltimer_ns();
	kh_stamp(KH_ST_FIN1);
	if (threadIdx.x == 0) { meta->finalize_us = (float)((tf1 - tf0) * 1e-3); meta->publish_us = 0.f; meta->entered_us = 0.f; meta->pad2 = 0u; }
	if (F.host_out) {
		__syncthreads();
		// the end of the kernel makes these stores visible to the host that synchronises on the stream: no system fence here
		const uint4 *src = reinterpret_cast<const uint4 *>(F.result_base);
		uint4 *dst = reinterpret_cast<uint4 *>(F.host_out);
		for (uint32_t i = threadIdx.x; i < F.result_bytes / 16; i += blockDim.x) dst[i] = __ldcg(src + i);
	}
	if (F0.clean_ptr) {
		// every other CTA has flushed and left (ticket), the join has read this rank's vector: keep the candidate partials
		// for apo_debug_partials and hand the next call a zeroed accumulator block
		__syncthreads();
		for (uint32_t i = threadIdx.x; i < (uint32_t)ACC_PER_CAND * F.C; i += blockDim.x) F0.snapshot[i] = __ldcg(F0.acc + i);
		__syncthreads();
		for (uint32_t i = threadIdx.x; i < F0.clean_words; i += blockDim.x) F0.clean_ptr[i] = 0ll;
	}
	if (F.host_out && threadIdx.x == 0) {
		// the timer of this last step lands in the host copy only (the device block was already copied out)
		reinterpret_cast<ResultMeta *>(F.host_out + F.meta_off)->publish_us = (float)((globaltimer_ns() - tf1) * 1e-3);
	}
	kh_stamp(KH_ST_PUBLISH);
}

}  // namespace apo
