// apo_kernels.h — host-visible launch interface of apo_kernels.cu (internal, not the ABI).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "../../include/apo_b200.h"

namespace apo {

struct Weights { double w[APO_NDIM]; };

// Cross-rank join of the packed int64 partial vector over NVLink peer memory (one process per GPU; SURVEY 8e).
// Every rank owns one peer-mapped block: two export slots (epoch parity) and one arrival flag per source rank.
// The CTA that finalises a scoring call publishes this rank's partials into its own slot, raises its flag in
// every peer's block, waits for all flags of the epoch in its OWN block (local polling), then sums the peers'
// slots with direct NVLink loads.  Integer sums: the result is the same on every rank and for every rank count.
constexpr int PEER_MAX = 8;
struct JoinParams {
	int nranks, rank;                       // nranks <= 1: no join
	uint32_t words;                         // int64 words exchanged (acc_words(C, nranks))
	uint32_t pad;
	unsigned long long epoch;               // > 0, identical on every rank for the same call
	long long *slot[PEER_MAX];              // export slot of rank r for this epoch's parity (peer-mapped address)
	unsigned long long *flag[PEER_MAX];     // arrival flags inside rank r's block: flag[r][source rank]
	long long *joined;                      // local: the summed vector
};

struct FinalizeParams {
	const long long *acc;
	uint32_t C, K;
	int nranks;
	int with_corpus;
	JoinParams join;
	uint8_t *result_base;       // device result block (scores | counts | topk | report | meta)
	uint8_t *host_out;          // page-locked, device-mapped copy of the block written by the finalising CTA; NULL = the host copies
	uint32_t result_bytes;
	uint32_t meta_off;          // ResultMeta inside the block
	// self-cleaning (one-shot calls): after the result is out, the finalising CTA keeps a copy of this rank's candidate
	// partials (apo_debug_partials) and zeroes the whole accumulator block, so the NEXT call needs no memset: one launch per call
	long long *clean_ptr;       // NULL = leave the accumulators alone (sessions)
	uint32_t clean_words;
	long long *snapshot;        // [4*C] copy of the candidate partials taken before cleaning
	double *scores;             // [C]
	uint64_t *counts;           // [C]
	unsigned long long *keys;   // [C] scratch
	unsigned long long *sel_key;// [K] scratch
	int32_t *sel_idx;           // [K] scratch
	int32_t *topk;              // [K]
	apo_corpus_report *report;
};

struct ResultMeta {             // tail of the result block
	uint32_t status;            // 0 ok, 1 = peer join timed out (a rank never arrived)
	uint32_t pad;
	float join_wait_us;         // publish -> all ranks arrived (includes the skew between ranks)
	float join_reduce_us;       // reading and summing the peers' slots
	float finalize_us;          // segmented sum + report + radix top-K (device timer, finalising CTA)
	float publish_us;           // result block -> caller's buffer, accumulators re-armed
	float entered_us;           // kernel start of the finalising CTA -> it entered the tail (its share of the scoring / scanning work)
	uint32_t pad2;
};

struct K2Params {
	const apo_record *recs;
	uint64_t T;
	uint64_t idx_base;
	uint32_t C;
	int rank;
	long long *acc;
	unsigned long long *ex_scratch;  // [18], preset to ~0
	unsigned int *ticket;            // preset to 0
	const double *lut;
	Weights W;
	int fuse_finalize;
	FinalizeParams fin;
};

struct K1Params {
	const uint8_t *base;        // first evaluation of candidate 0 inside the window
	uint64_t pitch_bytes;       // candidate row pitch
	uint32_t C;
	uint32_t tiles_per_cand;    // filled by run_reward9
	uint64_t T;                 // evaluations per candidate in this launch
	uint64_t total_tiles;       // filled by run_reward9
	uint32_t tune;              // experiments only (APO_K1_TUNE): bit0 no L2 hint, bits 1-3 log2 of bulk copies per stage
	long long *acc;             // accumulator vector (see apo_device.cuh)
	const double *lut;          // [0,512) total weight per presence mask, [512,1024) its reciprocal,
	                            // [1024,1088) categorical product table (apo_device.cuh CAT_*)
	Weights W;
	int corpus_on;              // run the corpus scan (K2) on one extra warp per CTA and the K2 tail in this launch
	K2Params corpus;
	uint32_t *bad;              // Form D: set to 1 when an evaluation's finalReward is outside [-512, 512) (fx_out_of_domain)
};


// Form Q (apo_compact.cu): 8 one-byte codes + fp32 d2 per evaluation
struct KqParams {
	const unsigned long long *q8;   // [C][pitch] codes, window base of candidate 0
	const float *d2;                // [C][pitch]  (0.0 when absent)
	const unsigned short *li;       // [C][pitch]  rotated presence-mask index into the LUT
	uint64_t pitch_evals;
	uint32_t C;
	uint32_t tiles_per_cand;
	uint64_t T;
	uint64_t total_tiles;
	long long *acc;
	const double *lut;              // as K1Params::lut
	const double *ptab;             // [8][256] value*weight per code (code 255 -> +0.0), table 0 = fl(0 + d0*w0)
	double w2;
	// mixed-lookup variants (0, 5, 6): table 0+1 fused into one exact prefix table, the first NF of the
	// six remaining coded dimensions read the fp32 value and multiply on the fp64 pipe instead
	const double *pair;             // [(n0+1)][(n1+1)] fl(fl(0 + d0*w0) + d1*w1); last row / column = absent
	const float *cbf;               // [8][256] code -> fp32 value (unused / absent -> 0.0f)
	uint32_t n0, n1;                // used codes of dimensions 0 and 1
	double wq[8];                   // weight of coded dimension j (push order 0,1,3..8)
	int corpus_on;                  // as K1Params
	K2Params corpus;
	uint32_t *bad;                  // as K1Params
	// Form W (the 8-byte copy of a resident Form D tensor): one word per evaluation, eight 4-bit dense codes (15 = absent) in
	// bits 0-31 and the fp32 tool_success_rate bit pattern in bits 32-63 (0x7FC00000 = absent).  Non-NULL: K1q reads this
	// instead of q8 / d2 / li, with the mixed-lookup tables above.
	const unsigned long long *qw;
};
// ---- categorical product table layout (built by apo_abi.cu build_luts, read by the kernels)
constexpr int CAT_D01 = 0;    // [fb + 3*err + 6*ended] -> fl(fl(0 + d0*w0) + d1*w1)      (12)
constexpr int CAT_D3 = 12;    // thresholds met 0..3 -> {1,-0.2,-0.5,-1}*w3, [4] = 0       (5)
constexpr int CAT_D4 = 17;    // {1,0.3,-0.3,-0.8}*w4                                      (5)
constexpr int CAT_D5 = 22;    // {1,0.5,0,-0.5}*w5                                         (5)
constexpr int CAT_D6 = 27;    // k = clamp(llm - thr, 0, 5) -> max(-1, 1 - k*0.4)*w6, [6] = 0 (7)
constexpr int CAT_D7 = 34;    // {1,0.5,0,-0.5}*w7                                         (5)
constexpr int CAT_D8 = 39;    // {1,0.3,-0.3,-0.8}*w8                                      (5)
// Direct tables for K1r: four dimensions depend on one small counter and the mode only, so the
// product is read straight from [agent][min(counter, cap)] — no threshold selects, no compares.
// Entries are copies of the level products above (same bits); slot "absent" holds +0.0.
constexpr int DIR_D3 = 64;    // [2][7]  min(toolFail, 5); slot 6 = no tool calls                 (TCS:701-708)
constexpr int DIR_D4 = 78;    // [2][27] min(toolCalls, 26); 0 = absent                            (TCS:711-718)
constexpr int DIR_D6 = 132;   // [2][10] min(llmCalls, 9); 0 = absent                              (TCS:733-737)
constexpr int DIR_D8 = 152;   // [2][11] min(turns, 10); 0 = absent                                (TCS:752-762)
constexpr int CAT_WORDS = 176;

constexpr int KQ_PAIR_MAX = 1024;   // entries of the prefix table that fit its shared-memory slot
constexpr uint32_t KW_D2_ABSENT = 0x7FC00000u;   // Form W: the one NaN pattern of an absent tool_success_rate
int kq_tile_evals(int variant);
int kw_tile_evals();                // K1q on Form W
cudaError_t run_reward9q(KqParams P, int variant, bool recip, int sm_count, cudaStream_t st);
// Form Q planes with dense codes < 15 in every coded dimension -> Form W words
cudaError_t run_pack_w(const unsigned long long *q8, const float *d2, const unsigned short *li, uint64_t n, unsigned long long *qw, cudaStream_t st);
cudaError_t run_transcode(const float *dims, uint64_t pitch_in, uint32_t C, uint64_t T, unsigned long long *q8, float *d2,
                          uint64_t pitch_out, uint32_t *codebook, uint32_t *overflow, cudaStream_t st);
cudaError_t run_recode(unsigned long long *q8, float *d2, unsigned short *li, uint64_t n, const uint8_t *remap, cudaStream_t st);
// ok_lo / ok_hi: bit 16 j + c set when code c of coded dimension j names a value; *bad |= 1 when an evaluation names a slot
// that does not (empty or NaN), or a NaN tool_success_rate slot
cudaError_t run_unpack_p(const uint32_t *pc, const unsigned short *pd, uint64_t pitch_in, uint32_t C, uint64_t T, const float *d2book,
                         uint64_t ok_lo, uint64_t ok_hi, uint32_t *bad, unsigned long long *q8, float *d2, unsigned short *li,
                         uint64_t pitch_out, cudaStream_t st);
cudaError_t run_collect_d2(const float *d2, const unsigned short *li, uint64_t n, uint32_t *table, uint32_t *count, cudaStream_t st);
cudaError_t run_pack_p(const unsigned long long *q8, const float *d2, const unsigned short *li, uint64_t n, const uint32_t *d2book, uint32_t nbook,
                       uint32_t *pc, unsigned short *pd, uint32_t *bad, cudaStream_t st);
cudaError_t run_decode(const unsigned long long *q8, const float *d2, const unsigned short *li, uint64_t n, const uint32_t *codebook, float *out, cudaStream_t st);

// ---- Form T (csrc/apo_tuple.cu): every evaluation is a 24-bit index into a per-tensor dictionary of distinct
// evaluations; the reward of a dictionary entry is computed once (k_tuple_values), K1t sums table entries.
constexpr uint32_t KT_TUPLES_MAX = 0xFFFFFFu;      // dictionary entries addressable by lo16 | hi8 << 16
constexpr int KT_VALID_SHIFT = 58;                 // table entry = rint(finalReward * 2^52) + (counted << 58)
constexpr uint32_t KT_HOT_MAX = 24576;             // K1t serves table entries [0, KT_HOT_MAX) from shared memory (192 KB)
struct KtParams {
	const unsigned short *tl;       // [C][pitch] low 16 bits of the tuple index
	const unsigned char *th;        // [C][pitch] high 8 bits
	uint64_t pitch_evals;           // multiple of 8; tl / th 16-byte aligned
	uint32_t C;
	uint32_t tiles_per_cand;
	uint64_t T;
	uint64_t total_tiles;
	long long *acc;
	const long long *tval;          // [n_tuples + 1]; the last entry is the zero sentinel out-of-range indices are clamped to
	uint32_t n_tuples;
	uint32_t hot;                   // entries [0, hot) are served from shared memory
	uint32_t *bad;                  // bit 0: an index >= n_tuples was met
};
struct TupleValParams {
	const uint32_t *tb_pc;          // [n] Form P code word of the entry (eight 4-bit codes, 15 = absent)
	const unsigned short *tb_pd;    // [n] 12-bit tool_success_rate index (4095 = absent)
	uint32_t n;
	const double *ptab;             // [8][256] as KqParams::ptab, but NaN in empty slots
	const double *lut;              // as K1Params::lut
	const float *d2book;            // [4096]
	double w2;
	long long *tval;                // [n + 1] out
	uint32_t *bad;                  // bit 1: an entry is not representable (|reward| >= 2, or it names an empty or NaN slot of a codebook)
};
int kt_tile_evals();
cudaError_t run_tuple_values(const TupleValParams &P, bool recip, cudaStream_t st);
cudaError_t run_reward9t(KtParams P, int sm_count, cudaStream_t st);

// K1t2 (k_reward9t2): the Form T copy of a resident Form D tensor read from a 16-bit plane alone, 2 B per evaluation.  That
// plane (ts) holds SLOTS of a slot-ordered copy of the table, chosen at load so that the shared-memory gather of one warp
// instruction meets few bank conflicts:
//   entry e <  h         16 slots 16 e + k, one per bank pair k (8-byte slots, 16 bank pairs); which copy an evaluation names
//                        is chosen per half-warp instruction of K1t2 (k_slot_plane): apart from the bank pairs its single-slot
//                        lanes need, when the window starts on the 128-evaluation grid
//   zero slot 16 h       value 0, count 0
//   entry e in [h, end)  one slot e + 15 h + 1 (end <= 2^16 - 1 - 15 h: every slot fits 16 bits)
//   entry e >= end       the zero slot, and the evaluation is listed
// Every copy holds the same value, so the choice of copy never changes a result.  Two lists of evaluations are added after
// the stream from the entry-order table: the exceptions (index >= 2^16) and the evaluations of entries in [end, 2^16).  A list
// holds per row, sorted by position, {position in the row, full index}; xb[c][b] is the list offset of the first listed
// evaluation of row c at or after position b * KT_XBLOCK (b <= nblk: xb[c][nblk] = xb[c + 1][0] ends the row), so any window
// finds its evaluations without a search.
constexpr uint32_t KT_XBLOCK = 8192;
constexpr uint32_t KT_SLOT_REP = 16;              // slots of a replicated entry
constexpr uint32_t KT_SLOT_H = 512;               // replicated entries when the list of entries [end, 2^16) stays short
// [end, 2^16): the entries without a slot when h of them are replicated
inline uint32_t kt_slot_end(uint32_t n, uint32_t h) {
	const uint32_t e = 65535u - (KT_SLOT_REP - 1) * h;
	return n < e ? n : e;
}
struct Kt2Params {
	const unsigned short *ts;       // [C][pitch] slots, from the window start (a multiple of 8)
	uint64_t pitch_evals;           // multiple of 8; ts 16-byte aligned
	uint32_t C;
	uint32_t tiles_per_cand;
	uint64_t T;                     // evaluations of the window
	uint64_t first;                 // window start in the row: the lists' positions are absolute
	uint64_t total_tiles;
	long long *acc;
	const long long *sval;          // [n_slots] the table in slot order
	uint32_t n_slots;
	uint32_t hot;                   // slots [0, hot) are served from shared memory
	const long long *tval;          // [n_tuples + 1] the table in entry order; tval[n_tuples] = 0
	uint32_t n_tuples;
	uint32_t xb_pitch;              // blocks per row + 1
	const uint2 *xs;                // exceptions, or NULL: every index is below 2^16
	const uint32_t *xb;             // [C][xb_pitch] block index of xs
	const uint2 *ys;                // evaluations of entries [end, 2^16), or NULL: none
	const uint32_t *yb;             // [C][xb_pitch] block index of ys
};
int kt2_tile_evals();
cudaError_t run_reward9t2(Kt2Params P, int sm_count, cudaStream_t st);
// the list of tl / th [C][tpitch] (T evaluations per row, T < 2^32) of the evaluations whose index is >= 2^16 (lo >= 2^16:
// the exceptions) or in [lo, 2^16): xb [C][nblk + 1] (nblk = ceil(T / KT_XBLOCK)), then xs [xb[C - 1][nblk]].  The same bytes
// for every grid.
cudaError_t run_tx_build(const unsigned short *tl, const unsigned char *th, uint64_t tpitch, uint32_t C, uint64_t T, uint32_t lo,
                         uint32_t *xb, uint2 *xs, int sm_count, cudaStream_t st);
// the slot-order table sval [end + 15 h + 1] of the entry-order one
cudaError_t run_tuple_slots(const long long *tval, uint32_t h, uint32_t end, long long *sval, cudaStream_t st);
// the slot plane ts [C][tpitch] of tl / th (positions t >= T are left alone)
cudaError_t run_slot_plane(const unsigned short *tl, const unsigned char *th, uint64_t tpitch, uint32_t C, uint64_t T, uint32_t h,
                           uint32_t end, unsigned short *ts, cudaStream_t st);

// ---- corpus digest (apo_kernels.cu): what a scoring call's corpus report needs from a large resident corpus, built at load.
// Only a VALID record's reward key (its categorical slots and d2: CatIdx) reaches the weight-dependent words of the report, so
// those are sums over the distinct keys with their record counts; every other word does not depend on the weights at all.
// Entry = {d2 bit pattern, slots | count << CD_COUNT_SHIFT}, slots = i01 | i3 << 4 | i4 << 7 | i5 << 10 | i6 << 13 | i7 << 16
// | i8 << 19.  fixed: the corpus-block words [CORP_TALLY, CORP_NREC) (tallies, byMode, patterns, tool totals) followed by the
// 18 first-three slots (inverted indices, as ex_insert keeps them) of the load-time scan.
constexpr int CD_COUNT_SHIFT = 22;
constexpr int CD_FIXED = 27;                 // CORP_NREC - CORP_TALLY
constexpr int CD_WORDS = CD_FIXED + 18;
struct CorpusDigestParams {
	const ulonglong2 *ent;                   // [*n]
	const unsigned long long *n;             // entry count
	const long long *fixed;                  // [CD_WORDS]
	K2Params k2;                             // block, example scratch, ticket, tables, weights and tail of the call (recs unused)
};
// the keys of recs[0, T) into table {key} / cnt [slots] (cleared first); misc[0] = keys inserted, misc[1] = 1 once that exceeds
// cap (the pass then stops early), then the entries into ent [cap] and their number into misc[2] (none when misc[1] is set)
cudaError_t run_cd_build(const apo_record *recs, uint64_t T, const double *lut, ulonglong2 *table, unsigned long long *cnt, uint64_t slots,
                         uint64_t cap, unsigned long long *misc, ulonglong2 *ent, int sm_count, cudaStream_t st);
// the corpus words of one scoring call from the digest, then the tail (corpus_tail) as the stand-alone scan runs it; n_host:
// the entry count, sizes the grid
cudaError_t run_corpus_digest(const CorpusDigestParams &P, uint64_t n_host, int sm_count, cudaStream_t st);

// K1h (k_reward9th): whole rows of the Form T copy from per-row dictionary counts.  A row's score needs only how often each
// entry occurs in it: sum_t table[idx(c, t)] = sum_e count[c][e] * table[e], the same integer.  Per row c, pairs
// [off[c], off[c + 1]) hold its entries that occur (t < T only), ascending, as entry | count << KH_COUNT_SHIFT.  The bytes
// depend on tl / th and T alone.
constexpr int KH_COUNT_SHIFT = 20;                // entries below 2^20 (the copy's dictionary cap), counts below 2^44
struct KhParams {
	const unsigned long long *pairs;  // [nnz]
	const uint64_t *off;              // [C + 1]; off[0] = 0, off[C] = nnz
	uint32_t C;
	uint64_t nnz;
	long long *acc;
	const long long *tval;            // [n_tuples + 1] the table in entry order
	int corpus_on;                    // every CTA then runs the digest pass over its share of cd's entries and the tail
	CorpusDigestParams cd;            // (cd.fixed NULL: the tail alone, for a call without a corpus report)
	uint64_t cd_n;                    // the digest's entry count as the host holds it (0 with cd.fixed NULL): picks each CTA's pass
};
cudaError_t run_reward9th(const KhParams &P, int sm_count, cudaStream_t st);
// The counts of rows [0, R) of tl / th [R][tpitch] (evaluations t < T) into cnt [R][npitch] (npitch a multiple of 32, zeroed
// by the caller), then nz [R * nchunk + 1] (nchunk = ceil(npitch / 8192)): the exclusive scan of the non-zero counts of every
// (row, 8192-entry chunk); nz[R * nchunk] is their total.
cudaError_t run_th_count(const unsigned short *tl, const unsigned char *th, uint64_t tpitch, uint32_t R, uint64_t T, uint32_t npitch,
                         uint32_t *cnt, uint32_t *nz, int sm_count, cudaStream_t st);
// the pairs of those rows from cnt and nz, from pairs[base] on, and their offsets off[0, R] (base included)
cudaError_t run_th_write(const uint32_t *cnt, uint32_t R, uint32_t npitch, const uint32_t *nz, uint64_t base, unsigned long long *pairs,
                         uint64_t *off, int sm_count, cudaStream_t st);

// Form T built on the device from a resident tensor's Form W words or Form Q planes (apo_dims_tuples).  The key of an
// evaluation is its Form W word: eight 4-bit codes in the low half, the fp32 tool_success_rate bits (KW_D2_ABSENT = absent)
// in the high half; the host maps the high half to the d2book index afterwards.  Hash tables hold {key, value} pairs,
// TB_EMPTY = free (never a key: the high half of a key is a non-NaN value or KW_D2_ABSENT).
constexpr unsigned long long TB_EMPTY = ~0ull;
struct TbSource {
	const unsigned long long *qw;   // Form W words, or NULL: Form Q planes q8 / d2 / li
	const unsigned long long *q8;
	const float *d2;
	const unsigned short *li;
	uint64_t pitch;                 // row pitch in evaluations, a multiple of 8
	uint32_t C;
	uint64_t T;                     // evaluations t >= T of a row are pads and are neither counted nor looked up
};
cudaError_t run_tb_clear(unsigned long long *table, uint64_t slots, cudaStream_t st);
// table[slots] {key, count}: exact counts of the distinct keys; *nkeys = keys inserted, *over |= 1 once that exceeds cap
// (the pass then stops early)
cudaError_t run_tb_count(const TbSource &S, unsigned long long *table, uint64_t slots, uint64_t cap, unsigned long long *nkeys,
                         uint32_t *over, int sm_count, cudaStream_t st);
// the occupied slots of table as (key, count) pairs in any order; *n receives their number
cudaError_t run_tb_compact(const unsigned long long *table, uint64_t slots, unsigned long long *keys, unsigned long long *counts,
                           unsigned long long *n, cudaStream_t st);
// table[slots] {key, rank} of keys[0, n) (keys in rank order), into a cleared table
cudaError_t run_tb_insert(const unsigned long long *keys, uint32_t n, unsigned long long *table, uint64_t slots, cudaStream_t st);
// tl / th [C][tpitch] = rank of every evaluation's key; *bad = 1 when a key is not in the table
cudaError_t run_tb_index(const TbSource &S, const unsigned long long *keys, uint32_t n, const unsigned long long *table, uint64_t slots,
                         unsigned short *tl, unsigned char *th, uint64_t tpitch, uint32_t *bad, int sm_count, cudaStream_t st);

// ---- per-candidate breakdown (csrc/apo_cand.cu): a second pass over the evaluations a scoring call reads.
// Own integer buffer, never part of the scoring accumulator vector: [C][CB_INT] words (a later cross-rank join is one
// integer sum of this part) followed by the first-three 'bad' slots [nranks][C][3] (inverted indices as ex_insert keeps them)
// and one domain word (CandParams::dom).
constexpr int CB_DIM = 0;        // 9 x (l0, l1, l2, count): exact sum of rint(v * 2^52) over non-null evaluations where dim i is present
constexpr int CB_TALLY = 36;     // total, good, bad
constexpr int CB_INT = 39;
enum CandSource { CAND_DIMS = 0, CAND_REC32 = 1, CAND_REC16 = 2, CAND_Q = 3, CAND_T = 4, CAND_W = 5 };
// The evaluations every per-candidate pass reads: those of one scoring launch (its window, candidate offset and record positions)
struct CandEvals {
	uint32_t C;
	uint64_t T;                     // evaluations per candidate in this launch
	uint64_t idx_base;              // record position of evaluation 0 of this launch (window start / streamed chunk start)
	uint64_t pitch_evals;           // candidate row pitch in evaluations
	const uint8_t *rows;            // Form D (36 B) / R (32 B) / R16 (16 B): evaluation 0 of candidate 0
	const unsigned long long *q8;   // Form Q planes
	const float *d2;
	const unsigned short *li;
	const unsigned long long *qw;   // Form W words (KqParams::qw)
	const float *cbf;               // Form Q / W: [8][256] code -> fp32 value
	const unsigned short *tl;       // Form T planes + dictionary
	const unsigned char *th;
	const uint32_t *tb_pc;
	const unsigned short *tb_pd;
	uint32_t n_tuples;
	const float *tbook;             // Form T: [8][16] 4-bit code -> fp32 value
	const float *d2book;            // Form T: [4096] tool_success_rate values
	const double *lut;              // as K1Params::lut: [512] total weight (<= 0: finalReward null) | reciprocal | categorical products
};
struct CandParams {
	CandEvals src;
	long long *ints;                // [C][CB_INT] of candidate 0 of this launch
	unsigned long long *ex;         // [C][3] of candidate 0 of this launch
	unsigned int *dom;              // set to 1 when a counted evaluation has a present dimension with |v| >= 2048 (or NaN)
};
cudaError_t run_cand_breakdown(const CandParams &P, int source, int sm_count, cudaStream_t st);
// ints / ex: the whole buffer; partials: the scoring call's candidate accumulators (4 words per candidate)
cudaError_t run_cand_report(const long long *ints, const unsigned long long *ex, const long long *partials, uint32_t C,
                            apo_candidate_report *out, cudaStream_t st);

// ---- per-candidate corpus report (csrc/apo_cand.cu): the corpus scan run over every candidate's rollout records (Form R / R16).
// Own buffer, never part of the scoring accumulator vector: [C][CC_WORDS] blocks in the corpus-block layout (apo_device.cuh
// CORP_*), whose CORP_NREC the pass accumulates itself and whose 18 CORP_EX words hold the first-three slots as inverted
// indices (ex_insert keys, 0 = empty), followed by [C][CC_WORDS] scratch where the report kernel converts them to index + 1.
constexpr int CC_WORDS = 68 + 18;   // CORP_FIXED + one rank's 18 example slots
struct CandCorpusParams {
	CandEvals src;                  // Form R (32 B) / R16 (16 B) rows
	double w2;
	long long *blk;                 // [C][CC_WORDS] of candidate 0 of this launch
};
cudaError_t run_cand_corpus(const CandCorpusParams &P, int row, int sm_count, cudaStream_t st);
// blk: the whole buffer ([C][CC_WORDS] blocks, then the scratch)
cudaError_t run_cand_corpus_report(long long *blk, uint32_t C, apo_corpus_report *out, cudaStream_t st);

// ---- per-candidate extremes (csrc/apo_cand.cu): the 32 lowest and 32 highest finalRewards of every candidate.
// A key is 128 bits {order-preserving u64 of the binary64 finalReward (complemented for the highest list), record position},
// all ones = empty.  A list pair is CX_WORDS words: [2 lists: lowest, highest][32 keys ascending][value word, position word].
// Own buffer: [C][CX_WORDS] lists that persist through a call or session | [cand_ext_slots(sm_count, C)][CX_WORDS] segments,
// the runs of one launch's warps (warp w's run of candidate c in slot w + c).
constexpr int CX_WORDS = 2 * 32 * 2;
constexpr uint64_t CX_MAX_WARPS_PER_SM = 2048 / 32;   // the pass's grid never holds more warps than the SMs can host
inline uint64_t cand_ext_slots(int sm_count, uint32_t C) { return CX_MAX_WARPS_PER_SM * (uint64_t)sm_count + C; }
struct CandExtParams {
	CandEvals src;
	Weights W;
	unsigned long long *lists;      // [C][CX_WORDS] of candidate 0 of this launch
	unsigned long long *seg;        // segment slots of this launch
};
cudaError_t run_cand_extremes(const CandExtParams &P, int source, bool recip, int sm_count, cudaStream_t st);

// ---- per-candidate group scores (csrc/apo_cand.cu): every candidate's evaluations split by the label of their record.
// Own buffer [C][G][GR_WORDS]: l0, l1, l2, withReward (the scoring partials' layout: the exact sum of rint(fr * 2^52) is
// l2 * 2^64 + l1 * 2^32 + l0, every flush adding its signed sum's 32-bit limbs to l0 and l1 and the rest to l2, and
// run_carry_limbs bounding l0 and l1 across launches as it bounds the partials'), then total, good, bad and one unused word.
constexpr int GR_WORDS = 8;
constexpr int GR_TALLY = 4;
struct CandGroupParams {
	CandEvals src;
	Weights W;
	const uint8_t *labels;          // [labels T] group of every record position (src.idx_base + t)
	uint32_t G;                     // 1..APO_GROUPS_MAX
	long long *words;               // [C][G][GR_WORDS] of candidate 0 of this launch
};
cudaError_t run_cand_groups(const CandGroupParams &P, int source, bool recip, int sm_count, cudaStream_t st);
// words: the whole buffer of C candidates
cudaError_t run_cand_groups_report(const long long *words, uint32_t C, uint32_t G, apo_group_score *out, cudaStream_t st);

// ---- per-candidate reward spread (csrc/apo_cand.cu): the exact sum of squares of every candidate's terms rint(fr * 2^52).
// Own buffer [C][SP_WORDS]: S2 as an unsigned 192-bit integer, least significant word first.  n and S1 are the scoring
// call's own partials.
constexpr int SP_WORDS = 3;
struct CandSpreadParams {
	CandEvals src;
	Weights W;
	unsigned long long *words;      // [C][SP_WORDS] of candidate 0 of this launch
};
cudaError_t run_cand_spread(const CandSpreadParams &P, int source, bool recip, int sm_count, cudaStream_t st);
// words: the whole buffer; partials: the scoring call's candidate accumulators (4 words per candidate)
cudaError_t run_cand_spread_report(const unsigned long long *words, const long long *partials, uint32_t C, struct apo_candidate_spread *out,
                                   cudaStream_t st);

// ---- per-candidate paired comparison (csrc/apo_cand.cu): every candidate against its reference on the same record positions.
// Own buffer [C][PR_WORDS]: D1 = sum d (192-bit two's complement), D2 = sum d^2 (unsigned 192-bit), each least significant
// word first, then wins, losses, ties, candOnly, refOnly.  Every word takes whole 64-bit adds (carried atomics for the sums):
// nothing accumulates in 32-bit limbs, so the pair words need no limb carry.
constexpr int PR_WORDS = 11;
constexpr int PR_D1 = 0, PR_D2 = 3, PR_CNT = 6;
struct CandPairParams {
	CandEvals src;
	Weights W;
	const uint32_t *refs;           // [C] reference of candidate 0 of this launch onwards: an absolute index, or APO_PAIR_NONE
	uint32_t base;                  // absolute index of candidate 0 of this launch: the row of refs[c] is refs[c] - base
	unsigned long long *words;      // [C][PR_WORDS] of candidate 0 of this launch
};
cudaError_t run_cand_pairs(const CandPairParams &P, int source, bool recip, int sm_count, cudaStream_t st);
// words / refs: the whole buffers of C candidates
cudaError_t run_cand_pair_report(const unsigned long long *words, const uint32_t *refs, uint32_t C, struct apo_candidate_pair *out,
                                 cudaStream_t st);

// ---- per-candidate paired comparison per record group (csrc/apo_cand.cu): the paired comparison restricted to the record
// positions of each label.  Own buffer [C][G][PR_WORDS], each (c, g) in the pair words' layout; no limb carry, as for them.
struct CandGroupPairParams {
	CandEvals src;
	Weights W;
	const uint8_t *labels;          // [labels T] group of every record position (src.idx_base + t)
	uint32_t G;                     // 1..APO_GROUPS_MAX
	const uint32_t *refs;           // as CandPairParams
	uint32_t base;
	unsigned long long *words;      // [C][G][PR_WORDS] of candidate 0 of this launch
};
cudaError_t run_cand_group_pairs(const CandGroupPairParams &P, int source, bool recip, int sm_count, cudaStream_t st);
// words / refs: the whole buffers of C candidates
cudaError_t run_cand_group_pairs_report(const unsigned long long *words, const uint32_t *refs, uint32_t C, uint32_t G,
                                        struct apo_candidate_pair *out, cudaStream_t st);

// ---- limb carry (csrc/apo_cand.cu): the (l0, l1, l2) triples that accumulate across the launches of a session or of a
// host-streaming call (the candidate partials, the breakdown's dimension words, the group words, the per-candidate corpus
// blocks' reward and dimension words) stay exact while l0 and l1 < 2^63.  limb_flush_bound: the most flushes one launch over
// `count` evaluations per candidate adds into one candidate's triple; LIMB_FLUSH_MAX: the most flushes a triple takes after
// run_carry_limbs has rewritten it (every triple w + r * row_words + first + 4 k, r < rows, k < per_row) to l0, l1 < 2^32.
constexpr uint64_t LIMB_FLUSH_MAX = (1ull << 26) - 1;
uint64_t limb_flush_bound(uint64_t count, int sm_count);
cudaError_t run_carry_limbs(long long *w, uint64_t rows, uint32_t row_words, uint32_t first, uint32_t per_row, cudaStream_t st);

int k1_tile_evals(int row, int variant);
cudaError_t run_reward9(K1Params P, int row, int variant, bool recip, int sm_count, cudaStream_t st);
cudaError_t run_detect6(const K2Params &P, int sm_count, cudaStream_t st);
cudaError_t run_finalize(const FinalizeParams &F, cudaStream_t st);
cudaError_t run_gen_dims(float *out, uint64_t pitch_evals, uint64_t seed, uint32_t c0, uint32_t C, uint64_t t0, uint64_t T,
                         uint32_t agent_permille, cudaStream_t st);
cudaError_t run_gen_records(apo_record *out, uint64_t pitch, uint64_t seed, uint32_t stream, uint32_t c0, uint32_t C,
                            uint64_t t0, uint64_t T, uint32_t agent_permille, cudaStream_t st);
cudaError_t run_gen_records16(apo_record16 *out, uint64_t pitch, uint64_t seed, uint32_t stream, uint32_t c0, uint32_t C,
                              uint64_t t0, uint64_t T, uint32_t agent_permille, cudaStream_t st);
cudaError_t run_touch(const void *p, uint64_t bytes, void *sink, cudaStream_t st);
cudaError_t run_fill_durclass(void *rows, uint32_t row_bytes, uint64_t n, cudaStream_t st);
cudaError_t run_reward_batch(const apo_record *recs, uint64_t n, const Weights &W, const double *lut, double *dims,
                             uint32_t *masks, double *finals, cudaStream_t st);

}  // namespace apo
