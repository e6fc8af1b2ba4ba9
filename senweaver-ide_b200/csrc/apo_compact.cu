// apo_compact.cu — Form Q: a lossless compact HBM layout for resident evaluations, and K1q.
//
// The path is HBM-bound (36 B per evaluation in Form D).  Eight of the nine reward dimensions
// of the reference take a handful of values (TCS:677-761: user_feedback, task_completion,
// tool_call_reliability, tool_call_efficiency, tool_duration_efficiency, response_efficiency,
// token_efficiency, conversation_efficiency); only tool_success_rate (d2 = succ/total*2-1,
// TCS:698) is a ratio.  Form Q therefore keeps, per evaluation,
//     q8  : 8 one-byte codes (dims 0,1,3,4,5,6,7,8; 255 = dimension absent)       8 B
//     d2  : the fp32 value of dim 2 (0.0 when absent)                              4 B
//     li  : the presence mask of the evaluation as a (bank-rotated) LUT index      2 B
// = 14 B instead of 36 B, plus one codebook of <= 255 fp32 bit patterns per coded dimension.
// The transcoder (k_transcode) builds the codebooks with a find-or-insert hash and refuses
// data with more than 255 distinct values in a coded dimension — the engine then simply keeps
// Form D.  It is lossless: decoding returns the original fp32 bit patterns (absent = NaN).
//
// K1q reads value*weight straight from a shared-memory product table indexed by code (built on
// the host with the same IEEE multiplications as TCS:781), so a coded dimension costs one LDS.64
// and one DADD; sums, division and the exact fixed-point accumulation are those of K1, hence the
// integer partial sums are bit-identical to K1's and to the oracle's.
//
// Form W is the 8-byte variant of the copy the engine keeps of a resident Form D tensor (apo_abi.cu build_twin) when every
// coded dimension takes at most 15 values: one word per evaluation, the eight dense codes as nibbles (15 = absent) and the
// fp32 d2 bits (KW_D2_ABSENT = absent).  K1q reads it with one bulk copy per tile and derives the LUT entry from the nibbles.
#include <cstdlib>
#include "apo_device.cuh"
#include "apo_kernels.h"
#include "apo_corpus.cuh"

namespace apo {

// dims held as codes, in byte order of q8: 0,1,3,4,5,6,7,8 (byte j <-> dim j < 2 ? j : j + 1)
constexpr uint32_t SLOT_EMPTY = 0xFFFFFFFFu;     // an fp32 NaN pattern: never a stored value

// =================================================================== transcoder Form D -> Form Q
// codebook: [8][256] uint32 (fp32 bit patterns, SLOT_EMPTY = free; slot 255 is never used),
// overflow: [8] flags.  Slots are only ever filled, never moved: a code handed out stays valid.
__device__ __forceinline__ uint32_t find_or_insert(uint32_t *s_slots, uint32_t *g_slots, uint32_t bits, uint32_t *overflow) {
	uint32_t h = (bits * 2654435761u) >> 24;                 // 0..255
	if (h == 255) h = 0;
	for (int probe = 0; probe < 255; probe++) {
		uint32_t cur = atomicOr(&s_slots[h], 0u);                // atomic read of this CTA's copy (slots only go EMPTY -> value)
		if (cur == bits) return h;
		if (cur == SLOT_EMPTY) {
			// not in this CTA's copy: consult / claim the global slot, then publish the global truth locally
			cur = atomicCAS(&g_slots[h], SLOT_EMPTY, bits);
			if (cur == SLOT_EMPTY) cur = bits;
			atomicAnd(&s_slots[h], cur);                             // EMPTY is all ones: AND installs the value, idempotent
			if (cur == bits) return h;
		}
		h = h == 254 ? 0 : h + 1;
	}
	*overflow = 1u;
	return 0;
}

__global__ void __launch_bounds__(256)
k_transcode(const float *dims, uint64_t pitch_in, uint32_t C, uint64_t T, unsigned long long *q8, float *d2,
            uint64_t pitch_out, uint32_t *codebook, uint32_t *overflow) {
	__shared__ uint32_t s_slots[8 * 256];
	for (int i = threadIdx.x; i < 8 * 256; i += blockDim.x) s_slots[i] = ((volatile uint32_t *)codebook)[i];
	__syncthreads();
	const uint32_t c = blockIdx.y;
	if (c >= C) return;
	for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < T; t += (uint64_t)gridDim.x * blockDim.x) {
		const float *row = dims + ((uint64_t)c * pitch_in + t) * APO_NDIM;
		unsigned long long q = 0;
#pragma unroll
		for (int j = 0; j < 8; j++) {
			const int dim = j < 2 ? j : j + 1;
			const float f = row[dim];
			uint32_t code = 255u;
			if (f == f) code = find_or_insert(s_slots + 256 * j, codebook + 256 * j, __float_as_uint(f), overflow + j);
			q |= (unsigned long long)code << (8 * j);
		}
		q8[(uint64_t)c * pitch_out + t] = q;
		const float f2 = row[2];
		d2[(uint64_t)c * pitch_out + t] = (f2 == f2) ? f2 : __int_as_float(0x7fc00000);
	}
}

cudaError_t run_transcode(const float *dims, uint64_t pitch_in, uint32_t C, uint64_t T, unsigned long long *q8, float *d2,
                          uint64_t pitch_out, uint32_t *codebook, uint32_t *overflow, cudaStream_t st) {
	if (C == 0 || T == 0) return cudaSuccess;
	uint64_t gx = (T + 255) / 256;
	if (gx > 132ull * 16) gx = 132ull * 16;
	for (uint32_t cb = 0; cb < C; cb += 32768) {
		const uint32_t cn = C - cb < 32768 ? C - cb : 32768;
		k_transcode<<<dim3((unsigned)gx, cn), 256, 0, st>>>(dims + (uint64_t)cb * pitch_in * APO_NDIM, pitch_in, cn, T,
		                                                   q8 + (uint64_t)cb * pitch_out, d2 + (uint64_t)cb * pitch_out, pitch_out, codebook, overflow);
	}
	return cudaGetLastError();
}

// Hash-slot codes -> dense codes (rank of the value inside its dimension), in place.  Dense codes
// keep the product-table entries of a dimension in adjacent shared-memory banks, so a warp whose
// lanes carry different codes reads them without bank conflicts (<= 16 values per dimension).
__global__ void __launch_bounds__(256)
k_recode(unsigned long long *q8, float *d2, unsigned short *li, uint64_t n, const uint8_t *remap /* [8][256] */) {
	__shared__ uint8_t s_map[8 * 256];
	for (int i = threadIdx.x; i < 8 * 256; i += blockDim.x) s_map[i] = remap[i];
	__syncthreads();
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
		const unsigned long long q = q8[i];
		unsigned long long o = 0;
		uint32_t mask = 0;                                   // natural presence mask, bit = dimension
#pragma unroll
		for (int j = 0; j < 8; j++) {
			const uint32_t c = s_map[256 * j + ((uint32_t)(q >> (8 * j)) & 255u)];
			o |= (unsigned long long)c << (8 * j);
			mask |= (c != 255u ? 1u : 0u) << (j < 2 ? j : j + 1);
		}
		const float f2 = d2[i];
		const bool p2 = (f2 == f2);
		mask |= (p2 ? 1u : 0u) << 2;
		q8[i] = o;
		d2[i] = p2 ? f2 : 0.0f;                               // +0.0 * w leaves the weighted sum unchanged
		li[i] = (unsigned short)lut_index(mask);
	}
}

cudaError_t run_recode(unsigned long long *q8, float *d2, unsigned short *li, uint64_t n, const uint8_t *remap, cudaStream_t st) {
	if (n == 0) return cudaSuccess;
	uint64_t g = (n + 255) / 256;
	if (g > 132ull * 32) g = 132ull * 32;
	k_recode<<<(unsigned)g, 256, 0, st>>>(q8, d2, li, n, remap);
	return cudaGetLastError();
}

// Form Q -> Form W (the 8-byte copy of a resident Form D tensor): the dense codes, every one < 15, as nibbles (255 -> 15)
// and the fp32 tool_success_rate bits, KW_D2_ABSENT when dimension 2 is absent.
__global__ void __launch_bounds__(256)
k_pack_w(const unsigned long long *q8, const float *d2, const unsigned short *li, uint64_t n, unsigned long long *qw) {
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
		const unsigned long long q = q8[i];
		uint32_t w = 0;
#pragma unroll
		for (int j = 0; j < 8; j++) w |= ((uint32_t)(q >> (8 * j)) & 15u) << (4 * j);     // 255 -> 15
		const uint32_t d = ((li[i] >> 6) & 1u) ? __float_as_uint(d2[i]) : KW_D2_ABSENT;     // rotated index: dim 2 lives in bit 6
		qw[i] = (unsigned long long)w | ((unsigned long long)d << 32);
	}
}

cudaError_t run_pack_w(const unsigned long long *q8, const float *d2, const unsigned short *li, uint64_t n, unsigned long long *qw, cudaStream_t st) {
	if (n == 0) return cudaSuccess;
	uint64_t g = (n + 255) / 256;
	if (g > 132ull * 32) g = 132ull * 32;
	k_pack_w<<<(unsigned)g, 256, 0, st>>>(q8, d2, li, n, qw);
	return cudaGetLastError();
}

// Form P -> Form Q on the device.  Form P is the tightest lossless wire format of the same evaluations for PCIe
// (6 B instead of 14 B / 36 B): the eight coded dimensions as 4-bit codes in one uint32 (15 = absent; needs <= 15 distinct
// values per dimension, true for dims produced by TCS:668-763) and tool_success_rate as a 12-bit index into a per-tensor
// fp32 table (4095 = absent; <= 4095 distinct ratios).  Expansion runs at HBM speed right behind the H2D copy of a window.
__global__ void __launch_bounds__(256)
k_unpack_p(const uint32_t *pc, const unsigned short *pd, uint64_t pitch_in, uint32_t C, uint64_t T, const float *d2book,
           uint64_t ok_lo, uint64_t ok_hi, uint32_t *bad, unsigned long long *q8, float *d2, unsigned short *li, uint64_t pitch_out) {
	// d2book is read through the read-only path: a tensor uses a few hundred of its 4096 entries, which stay in L1
	// (staging the 16 KB table in shared memory per block cost more than the block's own 256 evaluations)
	const uint32_t c = blockIdx.y;
	if (c >= C) return;
	bool named_empty = false;                // a code whose codebook slot is empty or NaN (ok bit 16 j + code clear), or a NaN d2
	for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < T; t += (uint64_t)gridDim.x * blockDim.x) {
		const uint32_t w = pc[(uint64_t)c * pitch_in + t];
		const uint32_t k2 = pd[(uint64_t)c * pitch_in + t] & 4095u;
		unsigned long long q = 0;
		uint32_t mask = 0;
#pragma unroll
		for (int j = 0; j < 8; j++) {
			const uint32_t nib = (w >> (4 * j)) & 15u;
			const uint32_t code = nib == 15u ? 255u : nib;
			q |= (unsigned long long)code << (8 * j);
			mask |= (nib != 15u ? 1u : 0u) << (j < 2 ? j : j + 1);
			if (nib != 15u && !(((j < 4 ? ok_lo : ok_hi) >> (16 * (j & 3) + nib)) & 1u)) named_empty = true;
		}
		const bool p2 = k2 != 4095u;
		mask |= (p2 ? 1u : 0u) << 2;
		const uint64_t o = (uint64_t)c * pitch_out + t;
		q8[o] = q;
		const float v2 = p2 ? __ldg(d2book + k2) : 0.0f;
		if (!(v2 == v2)) named_empty = true;
		d2[o] = v2;
		// The empty asm keeps the index computation in 32-bit registers.  Narrowed to 16-bit operations (the store is 16 bits
		// wide), ptxas for sm_90a dropped the dimension-2 presence bit, and K1q then renormalised without tool_success_rate.
		uint32_t idx = lut_index(mask);
		asm("" : "+r"(idx));
		li[o] = (unsigned short)idx;
	}
	if (named_empty) atomicOr(bad, 1u);
}

cudaError_t run_unpack_p(const uint32_t *pc, const unsigned short *pd, uint64_t pitch_in, uint32_t C, uint64_t T, const float *d2book,
                         uint64_t ok_lo, uint64_t ok_hi, uint32_t *bad, unsigned long long *q8, float *d2, unsigned short *li,
                         uint64_t pitch_out, cudaStream_t st) {
	if (C == 0 || T == 0) return cudaSuccess;
	uint64_t gx = (T + 1023) / 1024;                              // four evaluations per thread and row
	if (gx > 132ull * 8) gx = 132ull * 8;
	for (uint32_t cb = 0; cb < C; cb += 32768) {
		const uint32_t cn = C - cb < 32768 ? C - cb : 32768;
		k_unpack_p<<<dim3((unsigned)gx, cn), 256, 0, st>>>(pc + (uint64_t)cb * pitch_in, pd + (uint64_t)cb * pitch_in, pitch_in, cn, T, d2book,
		                                                 ok_lo, ok_hi, bad, q8 + (uint64_t)cb * pitch_out, d2 + (uint64_t)cb * pitch_out, li + (uint64_t)cb * pitch_out, pitch_out);
	}
	return cudaGetLastError();
}

// Form Q -> Form P (export of a resident tensor in the 6-byte wire format).  k_collect_d2 gathers the distinct
// tool_success_rate bit patterns into a 16384-slot open-addressing set; the host sorts them into the d2book; k_pack_p then
// writes the nibble word and the 12-bit index (binary search in the sorted book) per evaluation.
__global__ void __launch_bounds__(256)
k_collect_d2(const float *d2, const unsigned short *li, uint64_t n, uint32_t *table /* [16384], 0xFFFFFFFF = free */, uint32_t *count) {
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
		if (!((li[i] >> 6) & 1u)) continue;                       // rotated index: dimension 2 lives in bit 6
		const uint32_t bits = __float_as_uint(d2[i]);
		uint32_t h = (bits * 2654435761u) >> 18;
		for (int probe = 0; probe < 16384; probe++) {
			// look first: after the first few thousand evaluations every value is already there, and a plain (L1/L2) read of a
			// slot that only ever goes EMPTY -> value costs nothing next to 2.5 G contended atomics on a few hundred addresses
			uint32_t cur = *((volatile uint32_t *)&table[h]);
			if (cur == SLOT_EMPTY) {
				cur = atomicCAS(&table[h], SLOT_EMPTY, bits);
				if (cur == SLOT_EMPTY) { atomicAdd(count, 1u); break; }
			}
			if (cur == bits) break;
			h = (h + 1) & 16383u;
		}
	}
}

__device__ __forceinline__ bool d2_less(uint32_t x, uint32_t y) {     // by value, -0.0 before +0.0 (the host's sort order)
	const float fx = __uint_as_float(x), fy = __uint_as_float(y);
	return fx != fy ? fx < fy : x > y;
}

__global__ void __launch_bounds__(256)
k_pack_p(const unsigned long long *q8, const float *d2, const unsigned short *li, uint64_t n, const uint32_t *d2book, uint32_t nbook,
         uint32_t *pc, unsigned short *pd, uint32_t *bad) {
	__shared__ uint32_t s_book[4096];
	for (int i = threadIdx.x; i < 4096; i += blockDim.x) s_book[i] = d2book[i];
	__syncthreads();
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
		const unsigned long long q = q8[i];
		uint32_t w = 0;
#pragma unroll
		for (int j = 0; j < 8; j++) {
			const uint32_t code = (uint32_t)(q >> (8 * j)) & 255u;
			if (code != 255u && code > 14u) *bad = 1u;                // more than 15 distinct values: not representable
			w |= (code == 255u ? 15u : (code & 15u)) << (4 * j);
		}
		uint32_t k2 = 4095u;
		if ((li[i] >> 6) & 1u) {
			const uint32_t bits = __float_as_uint(d2[i]);
			uint32_t lo = 0, hi = nbook;                              // first entry not less than bits
			while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (d2_less(s_book[mid], bits)) lo = mid + 1; else hi = mid; }
			k2 = lo;
			if (lo >= nbook || s_book[lo] != bits) *bad = 1u;
		}
		pc[i] = w;
		pd[i] = (unsigned short)k2;
	}
}

cudaError_t run_collect_d2(const float *d2, const unsigned short *li, uint64_t n, uint32_t *table, uint32_t *count, cudaStream_t st) {
	if (n == 0) return cudaSuccess;
	uint64_t g = (n + 255) / 256;
	if (g > 132ull * 16) g = 132ull * 16;
	k_collect_d2<<<(unsigned)g, 256, 0, st>>>(d2, li, n, table, count);
	return cudaGetLastError();
}

cudaError_t run_pack_p(const unsigned long long *q8, const float *d2, const unsigned short *li, uint64_t n, const uint32_t *d2book, uint32_t nbook,
                       uint32_t *pc, unsigned short *pd, uint32_t *bad, cudaStream_t st) {
	if (n == 0) return cudaSuccess;
	uint64_t g = (n + 255) / 256;
	if (g > 132ull * 8) g = 132ull * 8;
	k_pack_p<<<(unsigned)g, 256, 0, st>>>(q8, d2, li, n, d2book, nbook, pc, pd, bad);
	return cudaGetLastError();
}

// Form Q -> Form D (tests, apo_dims_download)
__global__ void __launch_bounds__(256)
k_decode(const unsigned long long *q8, const float *d2, const unsigned short *li, uint64_t n, const uint32_t *codebook, float *out) {
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const unsigned long long q = q8[i];
	float *row = out + i * APO_NDIM;
#pragma unroll
	for (int j = 0; j < 8; j++) {
		const int dim = j < 2 ? j : j + 1;
		const uint32_t code = (uint32_t)(q >> (8 * j)) & 255u;
		row[dim] = code == 255u ? __int_as_float(0x7fc00000) : __uint_as_float(codebook[256 * j + code]);
	}
	row[2] = ((li[i] >> 6) & 1u) ? d2[i] : __int_as_float(0x7fc00000);     // rotated index: dim 2 lives in bit 6
}

cudaError_t run_decode(const unsigned long long *q8, const float *d2, const unsigned short *li, uint64_t n, const uint32_t *codebook, float *out, cudaStream_t st) {
	if (n == 0) return cudaSuccess;
	k_decode<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(q8, d2, li, n, codebook, out);
	return cudaGetLastError();
}

// =================================================================== K1q
struct QMeta { int32_t cand; int32_t n; };

// W: the stage holds Form W words (8 B per evaluation, one bulk copy) instead of the three Form Q planes (14 B, three copies),
// and the code tables live in the static KwTables (kw_tab) instead of the dynamic layout.
template <int CW, int EPT, int STAGES, bool W = false>
struct KqCfg {
	static constexpr int NCONS = CW * 32;
	static constexpr int TILE = NCONS * EPT;
	static constexpr int Q8_BYTES = TILE * 8, D2_BYTES = W ? 0 : TILE * 4, LI_BYTES = W ? 0 : TILE * 2;
	static constexpr int STAGE_BYTES = Q8_BYTES + D2_BYTES + LI_BYTES;
	static constexpr int LUT_OFF = STAGES * STAGE_BYTES;          // double2[512]
	static constexpr int PTAB_OFF = LUT_OFF + 512 * 16;           // double[8][256]
	static constexpr int CBF_OFF = PTAB_OFF + (W ? 0 : 8 * 256 * 8);        // float[8][256] code -> value (mixed-lookup variants)
	static constexpr int PAIR_OFF = CBF_OFF + (W ? 0 : 8 * 256 * 4);        // double[KQ_PAIR_MAX] exact prefix fl(fl(0 + d0*w0) + d1*w1)
	static constexpr int CAT_OFF = PAIR_OFF + (W ? 0 : KQ_PAIR_MAX * 8);    // categorical product table of the fused corpus scan
	static constexpr int BAR_OFF = CAT_OFF + CAT_WORDS * 8;
	static constexpr int META_OFF = BAR_OFF + 2 * STAGES * 8;
	static constexpr int EX_OFF = META_OFF + STAGES * 8;
	static constexpr int SMEM = EX_OFF + 18 * 8 + 16;
	static_assert(EPT % 4 == 0, "evaluations are processed in interleaved groups of four");
};

// byte j of a 32-bit word as one PRMT (the shift + mask form costs two ALU slots per table index)
template <int J>
__device__ __forceinline__ uint32_t byte_of(uint32_t w) {
	uint32_t r;
	asm("prmt.b32 %0, %1, 0, %2;" : "=r"(r) : "r"(w), "n"(0x4440 | J));
	return r;
}

// One Form-Q evaluation, first half: weighted sum in push order (TCS:777-783) + LUT entry.
__device__ __forceinline__ void evalq_ws(unsigned long long q, float d2f, uint32_t idx, const double *ptab, double w2,
                                         const double2 *lut, double &ws_out, double2 &t_out, uint32_t &valid) {
	const uint32_t lo = (uint32_t)q, hi = (uint32_t)(q >> 32);
	double ws = ptab[0 * 256 + byte_of<0>(lo)];                       // table 0 holds fl(0 + d0*w0)
	ws = __dadd_rn(ws, ptab[1 * 256 + byte_of<1>(lo)]);
	ws = __dadd_rn(ws, __dmul_rn((double)d2f, w2));                   // d2 is stored as +0.0 when absent
	ws = __dadd_rn(ws, ptab[2 * 256 + byte_of<2>(lo)]);
	ws = __dadd_rn(ws, ptab[3 * 256 + byte_of<3>(lo)]);
	ws = __dadd_rn(ws, ptab[4 * 256 + byte_of<0>(hi)]);
	ws = __dadd_rn(ws, ptab[5 * 256 + byte_of<1>(hi)]);
	ws = __dadd_rn(ws, ptab[6 * 256 + byte_of<2>(hi)]);
	ws = __dadd_rn(ws, ptab[7 * 256 + byte_of<3>(hi)]);
	ws_out = ws;
	t_out = lut[idx];                                                 // presence mask -> LUT index was fixed by the transcoder
	valid = t_out.x > 0.0 ? 1u : 0u;
}

// Mixed-lookup form of the same evaluation.  The 8-byte product reads of evalq_ws cost two shared-memory
// wavefronts each and that pipe is what bounds K1q; here dimensions 0 and 1 share one read of the exact
// prefix table, and NF of the other six read the 4-byte value (one wavefront) and form value*weight with
// the same F2F + DMUL the Form D kernel issues.  Every operation and its order are those of eval_ws.
template <int NF>
__device__ __forceinline__ void evalq_ws_mixed(unsigned long long q, float d2f, uint32_t idx, const double *ptab, const float *cbf,
                                               const double *pair, uint32_t n0, uint32_t n1, const double (&wq)[8], double w2,
                                               const double2 *lut, double &ws_out, double2 &t_out, uint32_t &valid) {
	const uint32_t lo = (uint32_t)q, hi = (uint32_t)(q >> 32);
	const uint32_t c0 = min(byte_of<0>(lo), n0), c1 = min(byte_of<1>(lo), n1);   // 255 (absent) -> last row / column
	double ws = pair[c0 * (n1 + 1u) + c1];
	ws = __dadd_rn(ws, __dmul_rn((double)d2f, w2));
#pragma unroll
	for (int j = 2; j < 8; j++) {
		const uint32_t code = j == 2 ? byte_of<2>(lo) : j == 3 ? byte_of<3>(lo) : j == 4 ? byte_of<0>(hi) : j == 5 ? byte_of<1>(hi)
		                      : j == 6 ? byte_of<2>(hi) : byte_of<3>(hi);
		if (j - 2 < NF) ws = __dadd_rn(ws, __dmul_rn((double)cbf[j * 256 + code], wq[j]));
		else ws = __dadd_rn(ws, ptab[j * 256 + code]);
	}
	ws_out = ws;
	t_out = lut[idx];
	valid = t_out.x > 0.0 ? 1u : 0u;
}

// Form W's code tables, in static shared memory.  ptab: value*weight by code for coded dimensions 2-7 (slot 15 = absent =
// +0.0), pair: the exact prefix fl(fl(0 + d0*w0) + d1*w1) indexed by the two low nibbles of a word, lut: double2[512]
// indexed by kw_key (the corpus warp keeps its own lut_index copy in the dynamic layout).  ptab comes first and the block is
// 256-byte aligned, so a product-table address is the block's address with its low byte replaced by 8 * code (kw_addr).
struct KwTables {
	double ptab[6][16];
	double pair[256];
	double2 lut[512];
};
__shared__ __align__(256) KwTables kw_tab;

// Form W's LUT order: the key the multiply-gather of evalw_ws yields.  Key bit r takes coded dimension 6 - 2r and bit r + 4
// coded dimension 7 - 2r (r = 0..3), bit 8 dimension 2: bits 0-2 hold dims 7, 5 and 3 (tokens, duration, tool use: the
// presences that vary in real data), so lanes with different masks mostly read different banks of an LDS.128 quarter-warp.
// natural_mask: bit = dimension; coded dimension k is dimension k < 2 ? k : k + 1.
__device__ __forceinline__ uint32_t kw_key(uint32_t natural_mask) {
	uint32_t key = ((natural_mask >> 2) & 1u) << 8;
#pragma unroll
	for (int r = 0; r < 4; r++) {
		const int lo = 6 - 2 * r, hi = 7 - 2 * r;                    // coded dimensions
		key |= ((natural_mask >> (lo < 2 ? lo : lo + 1)) & 1u) << r;
		key |= ((natural_mask >> (hi < 2 ? hi : hi + 1)) & 1u) << (r + 4);
	}
	return key;
}

// Slot of prefix entry i = c0 + 16 c1 (the low byte of a word): row c1, column c0 ^ 4 (c1 & 3).  Real data has <= 3 codes in
// dimension 0 and <= 4 in dimension 1; unswizzled, lanes with one c0 and different c1 would share a bank.
__device__ __forceinline__ uint32_t kw_pair_slot(uint32_t i) { return i ^ ((i >> 2) & 12u); }

// byte J of `offs` under the three high bytes of the 256-byte aligned shared address `base`: one PRMT, no add
template <int J>
__device__ __forceinline__ uint32_t kw_addr(uint32_t offs, uint32_t base) {
	uint32_t r;
	asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(offs), "r"(base), "n"(0x7650 | J));
	return r;
}

// Loads from the shared state space at a 32-bit address (smem_u32), so that a constant offset becomes the LDS immediate.
__device__ __forceinline__ double lds_f64(uint32_t a) {
	double v;
	asm("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(a));
	return v;
}
__device__ __forceinline__ double2 lds_f64x2(uint32_t a) {
	double2 v;
	asm("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "r"(a));
	return v;
}

// One Form W word: the operations and their order are those of evalq_ws_mixed with NF = 0 (prefix table, fl(d2*w2), the six
// other coded dimensions from product tables).  Integer work: the six product-table addresses come from two masked copies of
// the word, one PRMT each; the LUT entry from a carry test per nibble and one multiply-gather.  tab = smem_u32(&kw_tab).
__device__ __forceinline__ void evalw_ws(unsigned long long q, double w2, uint32_t tab, double &ws_out, double2 &t_out, uint32_t &valid) {
	constexpr uint32_t PAIR = offsetof(KwTables, pair), LUT = offsetof(KwTables, lut);
	const uint32_t w = (uint32_t)q;
	const float d2 = __uint_as_float((uint32_t)(q >> 32));
	const bool p2 = d2 == d2;                                         // absent = NaN
	const uint32_t ev = (w << 3) & 0x78787878u;                      // byte k: 8 * nibble 2k
	const uint32_t od = (w >> 1) & 0x78787878u;                      // byte k: 8 * nibble 2k + 1
	double ws = lds_f64(tab + PAIR + kw_pair_slot(w & 255u) * 8u);
	ws = __dadd_rn(ws, __dmul_rn((double)(p2 ? d2 : 0.0f), w2));    // +0.0 when absent, as Form Q stores it
	ws = __dadd_rn(ws, lds_f64(kw_addr<1>(ev, tab) + 0 * 128));      // coded dimension 2 = nibble 2
	ws = __dadd_rn(ws, lds_f64(kw_addr<1>(od, tab) + 1 * 128));
	ws = __dadd_rn(ws, lds_f64(kw_addr<2>(ev, tab) + 2 * 128));
	ws = __dadd_rn(ws, lds_f64(kw_addr<2>(od, tab) + 3 * 128));
	ws = __dadd_rn(ws, lds_f64(kw_addr<3>(ev, tab) + 4 * 128));
	ws = __dadd_rn(ws, lds_f64(kw_addr<3>(od, tab) + 5 * 128));
	ws_out = ws;
	// nibble k is 15 (absent) iff its low three bits carry into bit 3 on + 1 and bit 3 is set; present flags land on bits 4k
	const uint32_t pres = (~(((w & 0x77777777u) + 0x11111111u) & w) & 0x88888888u) >> 3;
	// bits 4k times 2^0 + 2^9 + 2^18 + 2^27 land on 64 distinct positions (no carries); bits 24-31 are the kw_key byte
	const uint32_t key8 = (pres * 0x08040201u) >> 24;
	t_out = lds_f64x2(key8 * 16u + (tab + LUT + (p2 ? 256u * 16u : 0u)));
	valid = t_out.x > 0.0 ? 1u : 0u;
}

template <int CW, int EPT, int STAGES, bool RECIP, int NF = -1, bool W = false>
__global__ void __launch_bounds__((CW + 2) * 32, 1)
k_reward9q(const KqParams P) {
	using Cfg = KqCfg<CW, EPT, STAGES, W>;
	static_assert(!W || NF == 0, "Form W runs the prefix-table form only");
	extern __shared__ __align__(128) uint8_t smem[];
	double2 *s_lut = reinterpret_cast<double2 *>(smem + Cfg::LUT_OFF);
	double *s_ptab = reinterpret_cast<double *>(smem + Cfg::PTAB_OFF);
	uint64_t *full = reinterpret_cast<uint64_t *>(smem + Cfg::BAR_OFF);
	uint64_t *empty = full + STAGES;
	QMeta *meta = reinterpret_cast<QMeta *>(smem + Cfg::META_OFF);
	double *s_cat = reinterpret_cast<double *>(smem + Cfg::CAT_OFF);
	float *s_cbf = reinterpret_cast<float *>(smem + Cfg::CBF_OFF);
	double *s_pair = reinterpret_cast<double *>(smem + Cfg::PAIR_OFF);
	unsigned long long *s_ex = reinterpret_cast<unsigned long long *>(smem + Cfg::EX_OFF);
	bool *s_last = reinterpret_cast<bool *>(smem + Cfg::EX_OFF + 18 * 8);

	const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
	for (int i = tid; i < 512; i += blockDim.x) s_lut[lut_index(i)] = make_double2(P.lut[i], P.lut[512 + i]);
	if constexpr (W) {
		// the host's [8][256] tables (dense codes < 15; slot 255 = absent = +0.0) cut to 16 slots, slot 15 = absent
		for (int i = tid; i < 512; i += blockDim.x) kw_tab.lut[kw_key(i)] = make_double2(P.lut[i], P.lut[512 + i]);
		for (int i = tid; i < 6 * 16; i += blockDim.x) kw_tab.ptab[i >> 4][i & 15] = P.ptab[((i >> 4) + 2) * 256 + ((i & 15) < 15 ? (i & 15) : 255)];
		for (int i = tid; i < 256; i += blockDim.x) {                  // [c1][c0]: index = the two low nibbles of a word
			const uint32_t c0 = min((uint32_t)i & 15u, P.n0), c1 = min((uint32_t)i >> 4, P.n1);
			kw_tab.pair[kw_pair_slot(i)] = P.pair[c0 * (P.n1 + 1u) + c1];
		}
	} else {
	for (int i = tid; i < 8 * 256; i += blockDim.x) s_ptab[i] = P.ptab[i];
	if (NF >= 0) {
		for (int i = tid; i < 8 * 256; i += blockDim.x) s_cbf[i] = P.cbf[i];
		for (int i = tid; i < (int)((P.n0 + 1u) * (P.n1 + 1u)); i += blockDim.x) s_pair[i] = P.pair[i];
	}
	}
	for (int i = tid; i < CAT_WORDS; i += blockDim.x) s_cat[i] = P.lut[1024 + i];
	if (tid == 0) {
		for (int s = 0; s < STAGES; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], CW); }
		mbar_fence_init();
	}
	__syncthreads();

	const uint64_t lo_t = P.total_tiles * blockIdx.x / gridDim.x;
	const uint64_t hi_t = P.total_tiles * (blockIdx.x + 1ull) / gridDim.x;

	if (warp == CW) {
		if (lane == 0) {
			const uint64_t pol = policy_evict_first();
			uint32_t it = 0;
			for (uint64_t tile = lo_t; tile <= hi_t; ++tile, ++it) {
				const int s = it % STAGES;
				const uint32_t ph = (it / STAGES) & 1u;
				mbar_wait(&empty[s], ph ^ 1u);
				if (tile == hi_t) { meta[s].cand = -1; meta[s].n = 0; mbar_arrive(&full[s]); break; }
				const uint32_t c = (uint32_t)(tile / P.tiles_per_cand);
				const uint64_t j = tile - (uint64_t)c * P.tiles_per_cand;
				const uint64_t e0 = j * Cfg::TILE;
				const uint64_t rem = P.T - e0;
				const uint32_t n = rem < (uint64_t)Cfg::TILE ? (uint32_t)rem : (uint32_t)Cfg::TILE;
				const uint32_t n8 = (n + 7u) & ~7u;                         // 64 / 32 / 16 B multiples for the three bulk copies
				meta[s].cand = (int32_t)c; meta[s].n = (int32_t)n;
				uint8_t *st = smem + s * Cfg::STAGE_BYTES;
				if constexpr (W) {
					mbar_expect_tx(&full[s], n8 * 8u);
					bulk_g2s(st, P.qw + (uint64_t)c * P.pitch_evals + e0, n8 * 8u, &full[s], pol);
				} else {
				mbar_expect_tx(&full[s], n8 * 14u);
				bulk_g2s(st, P.q8 + (uint64_t)c * P.pitch_evals + e0, n8 * 8u, &full[s], pol);
				bulk_g2s(st + Cfg::Q8_BYTES, P.d2 + (uint64_t)c * P.pitch_evals + e0, n8 * 4u, &full[s], pol);
				bulk_g2s(st + Cfg::Q8_BYTES + Cfg::D2_BYTES, P.li + (uint64_t)c * P.pitch_evals + e0, n8 * 2u, &full[s], pol);
				}
			}
		}
	} else if (warp == CW + 1) {
		if (P.corpus_on) {                                        // corpus warp: K2's scan on the spare issue slots
			if (lane < 18) s_ex[lane] = 0ull;
			__syncwarp();
			corpus_scan_warp<true>(P.corpus, (uint64_t)blockIdx.x * 32, (uint64_t)gridDim.x * 32, s_ex, s_cat, s_lut, lane);
		}
	} else {
	Acc128 acc; acc.zero();
	uint32_t cnt = 0;
	int cur = -1;
	uint32_t dom = 0;                                     // fx_domain_acc of every evaluation
	const double w2 = P.w2;
	double wq[8];
#pragma unroll
	for (int j = 0; j < 8; j++) wq[j] = P.wq[j];
	const uint32_t n0 = P.n0, n1 = P.n1;
	auto evalq = [&](unsigned long long q, float d2f, uint32_t idx, double &ws, double2 &t, uint32_t &ok) {
		if (NF >= 0) evalq_ws_mixed<(NF >= 0 ? NF : 0)>(q, d2f, idx, s_ptab, s_cbf, s_pair, n0, n1, wq, w2, s_lut, ws, t, ok);
		else evalq_ws(q, d2f, idx, s_ptab, w2, s_lut, ws, t, ok);
	};
	const uint32_t tab = smem_u32(&kw_tab);
	auto evalw = [&](unsigned long long q, double &ws, double2 &t, uint32_t &ok) { evalw_ws(q, w2, tab, ws, t, ok); };
	auto flush = [&](int c) {
		long long *dst = P.acc + (uint64_t)ACC_PER_CAND * c;
		flush_acc128(acc, dst, lane);
		const uint32_t n = warp_sum_u32(cnt);
		if (lane == 0 && n) atomicAdd((unsigned long long *)dst + 3, (unsigned long long)n);
		acc.zero(); cnt = 0;
	};

	for (uint32_t it = 0;; ++it) {
		const int s = it % STAGES;
		const uint32_t ph = (it / STAGES) & 1u;
		mbar_wait(&full[s], ph);
		const int c = meta[s].cand, n = meta[s].n;
		if (n == 0) break;
		if (c != cur) { if (cur >= 0) flush(cur); cur = c; }
		const unsigned long long *sq = reinterpret_cast<const unsigned long long *>(smem + s * Cfg::STAGE_BYTES);
		const float *sd = reinterpret_cast<const float *>(smem + s * Cfg::STAGE_BYTES + Cfg::Q8_BYTES);
		const unsigned short *sl = reinterpret_cast<const unsigned short *>(smem + s * Cfg::STAGE_BYTES + Cfg::Q8_BYTES + Cfg::D2_BYTES);
		if (n == Cfg::TILE) {
#pragma unroll
			for (int g = 0; g < EPT / 4; g++) {
				double ws4[4]; double2 t4[4];
#pragma unroll
				for (int k = 0; k < 4; k++) {
					const int e = (4 * g + k) * Cfg::NCONS + tid;              // 8 B / 4 B lane stride: conflict-free
					uint32_t ok;
					if constexpr (W) evalw(sq[e], ws4[k], t4[k], ok);
					else evalq(sq[e], sd[e], sl[e], ws4[k], t4[k], ok);
					cnt += ok;
				}
				const bool generic = !RECIP && ((__double2hiint(t4[0].y) | __double2hiint(t4[1].y) |
				                                 __double2hiint(t4[2].y) | __double2hiint(t4[3].y)) < 0);
				long long x4 = 0;
				if (!generic) {
#pragma unroll
					for (int k = 0; k < 4; k++) { const long long x = to_fx(div_fast<RECIP>(ws4[k], t4[k])); fx_domain_acc(dom, x); x4 += x; }
				} else {
#pragma unroll
					for (int k = 0; k < 4; k++) { const long long x = to_fx(div_lut<RECIP>(ws4[k], t4[k])); fx_domain_acc(dom, x); x4 += x; }
				}
				acc.add(x4);
			}
		} else {
			for (int k = 0; k < EPT; k++) {
				const int e = k * Cfg::NCONS + tid;
				if (e < n) {
					double ws; double2 t; uint32_t ok;
					if constexpr (W) evalw(sq[e], ws, t, ok);
					else evalq(sq[e], sd[e], sl[e], ws, t, ok);
					const long long x = to_fx(div_lut<RECIP>(ws, t));
					fx_domain_acc(dom, x);
					acc.add(x);
					cnt += ok;
				}
			}
		}
		__syncwarp();
		if (lane == 0) mbar_arrive(&empty[s]);
	}
	if (cur >= 0) flush(cur);
	if (fx_out_of_domain(dom)) *P.bad = 1u;               // read by the host after the call's synchronise
	}
	if (P.corpus_on) corpus_tail(P.corpus, s_ex, s_last, reinterpret_cast<unsigned long long *>(smem), 2048u);     // block-wide; stage 0 is free: scratch
}

template <int CW, int EPT, int STAGES, int NF = -1, bool W = false>
static cudaError_t launch_kq(const KqParams &P, int grid, bool recip, cudaStream_t st) {
	using Cfg = KqCfg<CW, EPT, STAGES, W>;
	cudaError_t err;
	if (recip) {
		auto k = k_reward9q<CW, EPT, STAGES, true, NF, W>;
		if ((err = allow_big_smem(k, Cfg::SMEM)) != cudaSuccess) return err;
		k<<<grid, (CW + 2) * 32, Cfg::SMEM, st>>>(P);
	} else {
		auto k = k_reward9q<CW, EPT, STAGES, false, NF, W>;
		if ((err = allow_big_smem(k, Cfg::SMEM)) != cudaSuccess) return err;
		k<<<grid, (CW + 2) * 32, Cfg::SMEM, st>>>(P);
	}
	return cudaGetLastError();
}

int kq_tile_evals(int variant) {
	switch (variant) {
	case 1: return KqCfg<16, 8, 3>::TILE;
	case 2: return KqCfg<24, 4, 4>::TILE;
	case 3: return KqCfg<20, 4, 5>::TILE;
	default: return KqCfg<20, 8, 2>::TILE;                       // 0 (mixed lookup, default), 4 (product tables only), 5, 6
	}
}

// Form W: 8 B per evaluation leave room for a deeper ring than Form Q's two 70 KB stages
constexpr int KW_CW = 20, KW_EPT = 8, KW_STAGES = 4;
int kw_tile_evals() { return KqCfg<KW_CW, KW_EPT, KW_STAGES, true>::TILE; }

cudaError_t run_reward9q(KqParams P, int variant, bool recip, int sm_count, cudaStream_t st) {
	const int tile = P.qw ? kw_tile_evals() : kq_tile_evals(variant);
	P.tiles_per_cand = (uint32_t)((P.T + tile - 1) / tile);
	P.total_tiles = (uint64_t)P.tiles_per_cand * P.C;
	if (P.total_tiles == 0) return cudaSuccess;
	int grid = sm_count;
	{ static const int env_grid = [] { const char *g = getenv("APO_K1_GRID"); return g ? atoi(g) : 0; }(); if (env_grid > 0 && env_grid < grid) grid = env_grid; }
	if ((uint64_t)grid > P.total_tiles) grid = (int)P.total_tiles;
	if (P.corpus_on && P.corpus.T) {
		const uint64_t want = (P.corpus.T + 63) / 64;
		const int more = (int)(want < (uint64_t)sm_count ? want : (uint64_t)sm_count);
		if (more > grid) grid = more;
	}
	// Form W: prefix table + the six other coded dimensions from product tables (NF = 0).  With 16-slot tables and one 8-byte
	// stage read, the fp32 reads of NF = 3 (Form Q's default) no longer pay for their F2F + DMUL: 5.62 against 5.33 ms per
	// flagship step on an H100 80GB HBM3 at 400 W (NF = 1: 5.48 / 5.97 ms)
	if (P.qw) return launch_kq<KW_CW, KW_EPT, KW_STAGES, 0, true>(P, grid, recip, st);
	switch (variant) {
	case 1: return launch_kq<16, 8, 3>(P, grid, recip, st);
	case 2: return launch_kq<24, 4, 4>(P, grid, recip, st);
	case 3: return launch_kq<20, 4, 5>(P, grid, recip, st);
	case 4: return launch_kq<20, 8, 2>(P, grid, recip, st);      // product tables only (also the fallback of 0)
	case 5: return launch_kq<20, 8, 2, 4>(P, grid, recip, st);   // prefix table + 4 fp32 dimensions
	case 6: return launch_kq<20, 8, 2, 6>(P, grid, recip, st);   // prefix table + all 6 through fp32
	default: return launch_kq<20, 8, 2, 3>(P, grid, recip, st);  // prefix table + 3 fp32 dimensions
	}
}

}  // namespace apo
