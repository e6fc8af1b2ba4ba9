// apo_abi.cu — the C ABI of libapo_b200.so (include/apo_b200.h): engine state, device
// memory ownership, launch sequencing, the NCCL join of record-axis shards.
//
// One engine = one GPU = one host thread at a time.  No CPU fallback anywhere: every
// compute entry point launches the sm_90a kernels of apo_kernels.cu or fails.
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <dlfcn.h>
#include <unistd.h>
#include <new>
#include <algorithm>
#include <string>
#include <utility>
#include <thread>
#include <vector>

#include "../../include/apo_b200.h"
#include "apo_format.h"
#include "apo_kernels.h"

namespace {

constexpr int ACC_PER_CAND = 4, CORP_FIXED = 68;
inline uint64_t acc_words(uint32_t C, int nranks) { return (uint64_t)ACC_PER_CAND * C + CORP_FIXED + 18ull * nranks; }

std::string g_create_error;

// TCS:766-776 in push order d0..d8
const double kDefaultWeights[APO_NDIM] = {0.25, 0.18, 0.12, 0.08, 0.05, 0.05, 0.08, 0.08, 0.11};
const int kCodedDim[8] = {0, 1, 3, 4, 5, 6, 7, 8};   // push-order dimension of coded dimension j (Form Q / P / T; d2 is not coded)

// ---- NCCL through dlopen: the library loads (and every single-GPU path works) without it
struct NcclId { char b[APO_UNIQUE_ID_BYTES]; };
struct NcclApi {
	void *h = nullptr;
	int (*GetUniqueId)(NcclId *) = nullptr;
	int (*CommInitRank)(void **, int, NcclId, int) = nullptr;
	int (*AllReduce)(const void *, void *, size_t, int, int, void *, cudaStream_t) = nullptr;
	int (*AllGather)(const void *, void *, size_t, int, void *, cudaStream_t) = nullptr;
	int (*CommDestroy)(void *) = nullptr;
	const char *(*GetErrorString)(int) = nullptr;
};
NcclApi g_nccl;
bool nccl_load(std::string &err) {
	if (g_nccl.h) return true;
	const char *names[] = {"libnccl.so.2", "libnccl.so"};
	for (const char *n : names) {
		g_nccl.h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
		if (g_nccl.h) break;
	}
	if (!g_nccl.h) { err = std::string("dlopen libnccl.so.2 failed: ") + dlerror(); return false; }
	g_nccl.GetUniqueId = (decltype(g_nccl.GetUniqueId))dlsym(g_nccl.h, "ncclGetUniqueId");
	g_nccl.CommInitRank = (decltype(g_nccl.CommInitRank))dlsym(g_nccl.h, "ncclCommInitRank");
	g_nccl.AllReduce = (decltype(g_nccl.AllReduce))dlsym(g_nccl.h, "ncclAllReduce");
	g_nccl.AllGather = (decltype(g_nccl.AllGather))dlsym(g_nccl.h, "ncclAllGather");
	g_nccl.CommDestroy = (decltype(g_nccl.CommDestroy))dlsym(g_nccl.h, "ncclCommDestroy");
	g_nccl.GetErrorString = (decltype(g_nccl.GetErrorString))dlsym(g_nccl.h, "ncclGetErrorString");
	if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllReduce || !g_nccl.CommDestroy) {
		err = "libnccl is missing a required symbol"; g_nccl.h = nullptr; return false;
	}
	return true;
}
constexpr int kNcclInt64 = 4, kNcclInt8 = 0, kNcclSum = 0, kNcclMin = 3;
constexpr uint32_t kMaxK = 16384;      // the K winners are ordered by counting (O(K^2)); beam widths are tiny (APO:288: 4)

template <class T>
struct DevBuf {
	T *p = nullptr; uint64_t cap = 0;   // capacity in elements
	cudaError_t reserve(uint64_t n) {
		if (n <= cap) return cudaSuccess;
		if (p) cudaFree(p);
		p = nullptr; cap = 0;
		cudaError_t e = cudaMalloc((void **)&p, n * sizeof(T));
		if (e == cudaSuccess) cap = n;
		return e;
	}
	void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

inline uint64_t round_up(uint64_t x, uint64_t m) { return (x + m - 1) / m * m; }

// K1q's lookup tables for one Form Q / P codebook under the weights of generation `gen` (load_qtables)
struct QTables {
	uint32_t book[8 * 256];
	DevBuf<double> ptab, pair; DevBuf<float> cbf;
	uint32_t n0 = 0, n1 = 0; bool pair_ok = false;
	uint64_t gen = 0;                        // apo_engine::weights_gen the tables were built for; 0: not built
	void release() { ptab.release(); pair.release(); cbf.release(); gen = 0; }
};

// Form T (csrc/apo_tuple.cu): a dictionary of distinct evaluations as Form P pairs, with its d2book and codebook
struct TupleDict {
	DevBuf<uint32_t> pc; DevBuf<unsigned short> pd; DevBuf<float> d2;
	uint32_t book[8 * 256]; uint32_t n = 0;
	void release() { pc.release(); pd.release(); d2.release(); }
};

// a resident Form T tensor: the dictionary and the [C][pitch] index planes
struct TupleTensor : TupleDict {
	DevBuf<unsigned short> l; DevBuf<unsigned char> h; uint32_t C = 0; uint64_t T = 0, pitch = 0;
	void unload() { C = 0; T = 0; n = 0; }
	void release() { TupleDict::release(); l.release(); h.release(); unload(); }
};

// A dictionary's table values rint(finalReward·2^52) (tuple_values).  Held (the Form T copy): val[recip] keeps the values of
// the current weights and ok[recip] says whether they are computed (0 not yet, 1 valid, 2 an entry is outside Form T's
// (-2, 2) domain).  Otherwise the values of one call in val[0], checked once it has synchronised (finish_score).
struct TupleVals {
	const bool held;
	DevBuf<double> ptab; DevBuf<long long> val[2]; DevBuf<uint32_t> bad;
	uint8_t ok[2] = {0, 0};
	explicit TupleVals(bool held = false) : held(held) {}
	long long *out(bool recip) const { return val[held && recip].p; }
	void release() { ptab.release(); val[0].release(); val[1].release(); bad.release(); ok[0] = ok[1] = 0; }
};

// The Form T copy of a large resident Form D tensor (build_twin_t), its held values and its exception list (build_twin_t2):
// t2 = K1t2 may read the copy from `l` alone; xs / xb hold the xn evaluations whose index is >= 2^16 and their block index.
struct TupleCopy : TupleTensor {
	TupleVals vals{true};
	DevBuf<uint2> xs; DevBuf<uint32_t> xb; uint64_t xn = 0; uint32_t nblk = 0; bool t2 = false;
	void release() { TupleTensor::release(); vals.release(); xs.release(); xb.release(); xn = 0; nblk = 0; t2 = false; }
};

}  // namespace

struct apo_engine {
	int device = 0, sm_count = 132;
	cudaStream_t own_stream = nullptr, stream = nullptr, copy_stream = nullptr;
	std::string err;
	apo::Weights W;
	double lut_tw[512], lut_rc[512], lut_cat[apo::CAT_WORDS];
	DevBuf<double> d_lut;          // [0,512) total weight, [512,1024) reciprocal, [1024,1088) categorical products

	DevBuf<apo_record> corpus; uint64_t corpus_T = 0, corpus_base = 0;
	DevBuf<float> dims; const float *dims_ptr = nullptr; uint32_t dims_C = 0; uint64_t dims_T = 0, dims_pitch = 0;
	// Form Q (compact) copy of the evaluations: replaces dims/dims_ptr when `compact` is set; when `twin` is set it sits beside
	// the engine's own fp32 tensor (built at load, a cache that is released whenever device memory runs short: see reserve)
	DevBuf<unsigned long long> q8; DevBuf<float> qd2; DevBuf<unsigned short> qli; DevBuf<uint32_t> qbook;   // qbook: [8][256] codebook + [8] overflow flags
	DevBuf<float> stage, d_d2book, d_d2stream;
	DevBuf<uint32_t> unpack_bad;                              // k_unpack_p: an evaluation named an empty or NaN codebook slot
	bool compact = false, twin = false;
	// K1q's tables: qt for the resident Form Q tensor or the Form Q / W copy (rebuilt by apo_set_weights), qt_stream for the
	// host-streaming Form Q / P calls (rebuilt by the next such call when its codebook or the weights changed)
	QTables qt, qt_stream; uint64_t weights_gen = 1;
	// twin_w: the copy is held as Form W words (qw, 8 B per evaluation; the Form Q planes are released) because no coded
	// dimension has more than 15 values
	DevBuf<unsigned long long> qw; bool twin_w = false;
	uint32_t d2book_host[4096]; uint32_t d2book_n = ~0u;       // Form P export of the resident tensor (~0 = not built yet)
	DevBuf<uint8_t> roll; uint32_t roll_C = 0, roll_row = 32; uint64_t roll_T = 0, roll_pitch = 0;   // Form R (32 B) or R16 (16 B) rows
	TupleTensor tup;                      // resident Form T (apo_tuples_upload / apo_dims_tuples)
	TupleDict tups;                       // the dictionary of a host-streaming Form T call
	TupleVals tvals;                      // the values a resident Form T launch or a host-streaming Form T call computes
	TupleVals *tvals_check = nullptr;     // the values the running call checks once it has synchronised
	TupleCopy tcopy;                      // the Form T copy of the fp32 tensor, released with its Form W / Q copy
	// apo_dims_tuples scratch (released when the build returns): hash table, (key, count) pairs / keys in rank order, counters
	DevBuf<unsigned long long> tb_table, tb_keys, tb_cnt, tb_misc;

	// acc: [acc_words(C, nranks)] partial vector | [18] example scratch (inverted indices) | [1] ticket — one allocation, so one
	// memset arms a scoring call.  acc_joined: the joined vector (> 1 rank); acc keeps this rank's partials.
	DevBuf<long long> acc, acc_joined, acc_snapshot; uint32_t last_C = 0;
	uint64_t acc_clean_words = 0;        // > 0: the first acc_clean_words of acc are known to be zero (left so by the last one-shot call)
	const long long *partials_src = nullptr;   // where apo_debug_partials finds the candidate partials of the last call
	DevBuf<unsigned long long> misc;     // NCCL warm-up / status scratch
	DevBuf<uint8_t> result;              // scores | counts | topk | report
	DevBuf<unsigned long long> keys, sel_key; DevBuf<int32_t> sel_idx;
	uint8_t *h_result = nullptr; uint64_t h_result_cap = 0;
	// page-locked, device-mapped word K1 (Form D) and K1q set when an evaluation's finalReward is outside [-512, 512): cleared
	// when a call or session begins, read after its synchronise (no extra copy or launch per call)
	volatile uint32_t *h_domain = nullptr;
	DevBuf<uint8_t> win[2]; cudaEvent_t win_free[2] = {nullptr, nullptr}, win_ready[2] = {nullptr, nullptr};
	uint8_t *h_stage[2] = {nullptr, nullptr}; uint64_t h_stage_cap = 0; cudaEvent_t stage_done[2] = {nullptr, nullptr};   // pinned staging of pageable callers
	DevBuf<apo_record> batch_in; DevBuf<double> batch_out; DevBuf<uint32_t> batch_mask;

	void *comm = nullptr; int nranks = 1, rank = 0;
	// peer-memory join (csrc/apo_corpus.cuh peer_join): this rank's block and the peer-mapped views of the others
	uint8_t *peer_block = nullptr; uint64_t peer_slot_words = 0; bool peer_ok = false;
	void *peer_base[apo::PEER_MAX] = {nullptr}; bool peer_ipc[apo::PEER_MAX] = {false};
	unsigned long long join_epoch = 0;
	bool env_no_fuse = false, env_force_fuse = false, env_no_staging = false, env_nccl_join = false, env_no_twin = false;   // apo_set_tuning
	bool env_no_twin_t = false, env_twin_t = false, env_no_twin_t2 = false;
	double stream_bytes_per_ms = 7.4e9, stream_q_bytes_per_ms = 5.0e9, stream_w_bytes_per_ms = 6.0e9, scan_ms_per_record = 3.35e-7;   // fuse heuristic, derived from the device at apo_create
	size_t mem_pitch_max = 0;
	uint8_t *zc_host = nullptr; uint64_t zc_cap = 0;   // zero-copy block of the single-trace path
	bool timing_on = true;
	cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
	std::vector<cudaEvent_t> k1_ev;      // start/stop pairs of the K1 launches of the current scoring call
	size_t k1_used = 0;
	uint32_t score_C = 0; bool scoring = false;
	apo_timing timing{};
	// per-candidate breakdown (APO_SCORE_CANDIDATES, csrc/apo_cand.cu): its own integers, never part of the accumulator vector
	DevBuf<long long> cand_acc;              // [C][CB_INT] integers | [C][3] first-three 'bad' slots | domain word
	DevBuf<apo_candidate_report> cand_rep;   // reports of the last flagged call
	DevBuf<float> cand_book;                 // Form T: [8][16] code -> fp32 value of the dictionary's codebook
	uint32_t cand_C = 0;
	bool cand_armed = false;                 // cand_acc zeroed for this call / session
	bool cand_every = true;                  // every accumulate of the session so far set the flag
	bool cand_ready = false;                 // cand_rep holds the breakdown of the last scoring call
	// per-candidate corpus report (APO_SCORE_CANDIDATE_CORPUS, csrc/apo_cand.cu k_cand_corpus): its own blocks, as cand_acc
	DevBuf<long long> ccorp_acc;             // [C][CC_WORDS] corpus blocks | [C][CC_WORDS] scratch of the report kernel
	DevBuf<apo_corpus_report> ccorp_rep;     // reports of the last flagged call
	uint32_t ccorp_C = 0;
	bool ccorp_armed = false, ccorp_every = true, ccorp_ready = false;   // as cand_armed / cand_every / cand_ready
};

namespace {

int fail(apo_engine *e, int code, const char *fmt, ...) {
	char buf[512];
	va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
	if (e) e->err = buf; else g_create_error = buf;
	return code;
}
#define CK(call)                                                                                    \
	do {                                                                                            \
		cudaError_t _c = (call);                                                                    \
		if (_c != cudaSuccess) return fail(e, APO_E_CUDA, "%s: %s (%s:%d)", #call, cudaGetErrorString(_c), __FILE__, __LINE__); \
	} while (0)

void drop_twin(apo_engine *e) {
	e->tcopy.release();
	if (!e->twin) return;
	e->q8.release(); e->qd2.release(); e->qli.release(); e->qw.release();
	e->twin = e->twin_w = false;
}

// Every engine buffer grows through here.  The Form Q / W / T copies of the fp32 tensor are a cache: an allocation that fails for lack
// of device memory while it is held releases it and is tried once more, so holding it never fails a call that would succeed
// without it.  Launches already queued may still read the copy: they finish first.  A resident call picks the evaluations
// it reads (route_twin) only after its last allocation before its launches.
template <class T>
cudaError_t reserve(apo_engine *e, DevBuf<T> &b, uint64_t n) {
	cudaError_t c = b.reserve(n);
	if (c != cudaErrorMemoryAllocation || !e->twin) return c;
	cudaGetLastError();
	if ((c = cudaStreamSynchronize(e->stream)) != cudaSuccess) return c;
	drop_twin(e);
	return b.reserve(n);
}

void build_luts(apo_engine *e) {
	for (uint32_t m = 0; m < 512; m++) {
		double tw = 0.0;                            // TCS:777-783: totalWeight += w in push order
		for (int i = 0; i < APO_NDIM; i++) if (m & (1u << i)) tw += e->W.w[i];
		if (!(tw > 0.0)) tw = -1.0;                 // totalWeight == 0: finalReward stays null (TCS:784); a negative entry tells the kernels not to count it
		e->lut_tw[m] = tw;
		// K1 divides by multiplying with RN(1/tw) + one FMA correction (Markstein); that is only
		// proven correctly rounded when the significand of tw is not all ones — flag those masks
		// with a negative reciprocal so the kernel takes the generic IEEE division for them.
		uint64_t bits; memcpy(&bits, &tw, 8);
		const bool all_ones = (bits & 0xFFFFFFFFFFFFFull) == 0xFFFFFFFFFFFFFull;
		e->lut_rc[m] = tw < 0.0 ? 1.0 : (all_ones ? -(1.0 / tw) : 1.0 / tw);
	}
	// categorical product table (csrc/apo_device.cuh CAT_*): value * weight with the same IEEE
	// multiplications the reference performs at TCS:781, tabulated once per weight vector
	const double *w = e->W.w;
	double *c = e->lut_cat;
	for (int i = 0; i < apo::CAT_WORDS; i++) c[i] = 0.0;
	for (int ended = 0; ended < 2; ended++)
		for (int err = 0; err < 2; err++)
			for (int fb = 0; fb < 3; fb++) {
				const double d0 = fb == 1 ? 1.0 : (fb == 2 ? -1.0 : 0.0);                       // TCS:677-678
				double d1 = 0.5;                                                                 // TCS:682-691
				if (ended && !err) d1 = 0.8;
				if (err) d1 = -0.5;
				if (fb == 1) d1 = 1.0;
				volatile double s = 0.0;
				s = s + d0 * w[0];
				s = s + d1 * w[1];
				c[0 + fb + 3 * err + 6 * ended] = s;
			}
	const double lv_rel[4] = {1.0, -0.2, -0.5, -1.0}, lv_cnt[4] = {1.0, 0.3, -0.3, -0.8}, lv_dur[4] = {1.0, 0.5, 0.0, -0.5};
	for (int k = 0; k < 4; k++) {
		c[12 + k] = lv_rel[k] * w[3]; c[17 + k] = lv_cnt[k] * w[4]; c[22 + k] = lv_dur[k] * w[5];
		c[34 + k] = lv_dur[k] * w[7]; c[39 + k] = lv_cnt[k] * w[8];
	}
	for (int k = 0; k < 6; k++) {
		volatile double over = (double)k;
		volatile double m = over * 0.4;
		double ef = 1 - m;                                                                       // TCS:735
		if (ef < -1) ef = -1;
		c[27 + k] = ef * w[6];
	}
	// direct tables of K1r: [agent][min(counter, cap)] -> the level product above (bit copies)
	using namespace apo;
	for (int ag = 0; ag < 2; ag++) {
		const uint32_t sev = ag ? 5u : 3u, mod = ag ? 3u : 2u, mnr = ag ? 2u : 1u;                       // TCS:702-704
		for (uint32_t f = 0; f <= 5; f++) c[DIR_D3 + ag * 7 + f] = c[CAT_D3 + (f >= mnr) + (f >= mod) + (f >= sev)];
		c[DIR_D3 + ag * 7 + 6] = 0.0;
		const uint32_t cexc = ag ? 8u : 3u, cgood = ag ? 15u : 6u, cfair = ag ? 25u : 10u;               // TCS:711-713
		c[DIR_D4 + ag * 27] = 0.0;
		for (uint32_t n = 1; n <= 26; n++) c[DIR_D4 + ag * 27 + n] = c[CAT_D4 + (n > cexc) + (n > cgood) + (n > cfair)];
		const uint32_t thr6 = ag ? 3u : 1u;                                                               // TCS:734
		c[DIR_D6 + ag * 10] = 0.0;
		for (uint32_t n = 1; n <= 9; n++) { const uint32_t over = n > thr6 ? n - thr6 : 0u; c[DIR_D6 + ag * 10 + n] = c[CAT_D6 + (over < 5u ? over : 5u)]; }
		const uint32_t thr8 = ag ? 3u : 2u;                                                               // TCS:756
		c[DIR_D8 + ag * 11] = 0.0;
		for (uint32_t n = 1; n <= 10; n++) c[DIR_D8 + ag * 11 + n] = c[CAT_D8 + (n > thr8) + (n > 2 * thr8) + (n > 3 * thr8)];
	}
}

int upload_luts(apo_engine *e) {
	CK(reserve(e, e->d_lut, 1024 + apo::CAT_WORDS));
	CK(cudaMemcpyAsync(e->d_lut.p + 1024, e->lut_cat, apo::CAT_WORDS * 8, cudaMemcpyHostToDevice, e->stream));
	CK(cudaMemcpyAsync(e->d_lut.p, e->lut_tw, 512 * 8, cudaMemcpyHostToDevice, e->stream));
	CK(cudaMemcpyAsync(e->d_lut.p + 512, e->lut_rc, 512 * 8, cudaMemcpyHostToDevice, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	return APO_OK;
}

// value*weight per code for the eight coded dimensions (csrc/apo_compact.cu); table 0 = fl(0 + d0*w0).  Empty slots hold
// `empty`: +0.0 for K1q, NaN for k_tuple_values, which refuses an entry that names one.  Slot 255 (absent) is +0.0.
std::vector<double> make_ptab(const uint32_t *book, const apo::Weights &W, double empty = 0.0) {
	std::vector<double> tab(8 * 256, 0.0);
	for (int j = 0; j < 8; j++)
		for (int c = 0; c < 255; c++) {
			const uint32_t bits = book[256 * j + c];
			if (bits == 0xFFFFFFFFu) { tab[256 * j + c] = empty; continue; }
			float f; memcpy(&f, &bits, 4);
			volatile double p = (double)f * W.w[kCodedDim[j]];          // TCS:781 value * weight
			if (j == 0) { volatile double z = 0.0; p = z + p; }          // weightedSum = 0 + first product
			tab[256 * j + c] = p;
		}
	return tab;
}

// q's tables for `book` under the current weights, rebuilt unless q already holds exactly those
int load_qtables(apo_engine *e, QTables &q, const uint32_t *book) {
	if (q.gen == e->weights_gen && memcmp(q.book, book, sizeof q.book) == 0) return APO_OK;
	q.gen = 0;                                                    // until the tables below are complete
	memmove(q.book, book, sizeof q.book);                         // apo_set_weights rebuilds q from its own book
	const std::vector<double> tab = make_ptab(q.book, e->W);
	CK(reserve(e, q.ptab, 8 * 256));
	CK(cudaMemcpyAsync(q.ptab.p, tab.data(), 8 * 256 * 8, cudaMemcpyHostToDevice, e->stream));
	// tables of the mixed-lookup variants: fp32 values per code, and the exact two-term prefix of dimensions 0 and 1
	std::vector<float> cbf(8 * 256, 0.0f);
	uint32_t used[8] = {0};
	for (int j = 0; j < 8; j++)
		for (int c = 0; c < 255; c++) {
			const uint32_t bits = q.book[256 * j + c];
			if (bits == 0xFFFFFFFFu) continue;
			memcpy(&cbf[256 * j + c], &bits, 4);
			used[j] = (uint32_t)c + 1;                                // dense codes: 0 .. used-1
		}
	q.n0 = used[0]; q.n1 = used[1];
	q.pair_ok = (uint64_t)(used[0] + 1) * (used[1] + 1) <= (uint64_t)apo::KQ_PAIR_MAX;
	std::vector<double> pair(apo::KQ_PAIR_MAX, 0.0);
	if (q.pair_ok)
		for (uint32_t a = 0; a <= used[0]; a++)
			for (uint32_t b = 0; b <= used[1]; b++) {
				volatile double s = tab[a < used[0] ? a : 255];           // fl(0 + d0*w0), +0.0 when absent
				s = s + tab[256 + (b < used[1] ? b : 255)];               // + d1*w1 (TCS:781, second push)
				pair[a * (used[1] + 1) + b] = s;
			}
	CK(reserve(e, q.cbf, 8 * 256));
	CK(reserve(e, q.pair, apo::KQ_PAIR_MAX));
	CK(cudaMemcpyAsync(q.cbf.p, cbf.data(), 8 * 256 * 4, cudaMemcpyHostToDevice, e->stream));
	CK(cudaMemcpyAsync(q.pair.p, pair.data(), apo::KQ_PAIR_MAX * 8, cudaMemcpyHostToDevice, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	q.gen = e->weights_gen;
	return APO_OK;
}

int compact_begin(apo_engine *e, uint32_t C, uint64_t pitch) {
	CK(reserve(e, e->q8, (uint64_t)(C ? C : 1) * pitch));
	CK(reserve(e, e->qd2, (uint64_t)(C ? C : 1) * pitch));
	CK(reserve(e, e->qli, (uint64_t)(C ? C : 1) * pitch));
	CK(reserve(e, e->qbook, 8 * 256 + 8));
	CK(cudaMemsetAsync(e->qbook.p, 0xFF, 8 * 256 * 4, e->stream));
	CK(cudaMemsetAsync(e->qbook.p + 8 * 256, 0, 8 * 4, e->stream));
	// pad evaluations of every row: all codes 255 + NaN = finalReward null
	CK(cudaMemsetAsync(e->q8.p, 0xFF, (uint64_t)(C ? C : 1) * pitch * 8, e->stream));
	CK(cudaMemsetAsync(e->qd2.p, 0xFF, (uint64_t)(C ? C : 1) * pitch * 4, e->stream));
	return APO_OK;
}

// returns APO_E_STATE when a coded dimension has more than 255 distinct values (twin: without an error text).  twin: the planes
// become the Form Q copy of the engine's fp32 tensor, which stays loaded; otherwise they replace it.
int compact_finish(apo_engine *e, uint32_t C, uint64_t T, uint64_t pitch, bool twin = false) {
	uint32_t host[8 * 256 + 8];
	CK(cudaMemcpyAsync(host, e->qbook.p, sizeof host, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	for (int j = 0; j < 8; j++)
		if (host[8 * 256 + j]) {
			e->q8.release(); e->qd2.release(); e->qli.release();
			if (twin) return APO_E_STATE;
			return fail(e, APO_E_STATE, "evaluations are not categorical: coded dimension %d has more than 255 distinct values; Form D is kept", j < 2 ? j : j + 1);
		}
	// hash-slot codes -> dense codes ordered by value (deterministic, bank-conflict-free table reads)
	uint8_t remap[8 * 256];
	uint32_t dense[8 * 256];
	for (int j = 0; j < 8; j++) {
		std::vector<std::pair<float, int>> used;
		for (int s = 0; s < 255; s++) {
			const uint32_t bits = host[256 * j + s];
			if (bits != 0xFFFFFFFFu) { float f; memcpy(&f, &bits, 4); used.push_back({f, s}); }
		}
		std::sort(used.begin(), used.end(), [&](const std::pair<float, int> &a, const std::pair<float, int> &b) {
			if (a.first != b.first) return a.first < b.first;
			return host[256 * j + a.second] > host[256 * j + b.second];      // -0.0 (sign bit set) before +0.0
		});
		for (int c = 0; c < 256; c++) { remap[256 * j + c] = 255; dense[256 * j + c] = 0xFFFFFFFFu; }
		for (size_t r = 0; r < used.size(); r++) { remap[256 * j + used[r].second] = (uint8_t)r; dense[256 * j + r] = host[256 * j + used[r].second]; }
	}
	CK(reserve(e, e->stage, 1024));
	CK(cudaMemcpyAsync(e->stage.p, remap, sizeof remap, cudaMemcpyHostToDevice, e->stream));
	CK(apo::run_recode(e->q8.p, e->qd2.p, e->qli.p, (uint64_t)C * pitch, (const uint8_t *)e->stage.p, e->stream));
	CK(cudaMemcpyAsync(e->qbook.p, dense, sizeof dense, cudaMemcpyHostToDevice, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	int rc = load_qtables(e, e->qt, dense);
	if (rc) return rc;
	if (twin) e->twin = true;
	else { e->compact = true; e->dims_C = C; e->dims_T = T; e->dims_pitch = pitch; e->dims_ptr = nullptr; }
	e->d2book_n = ~0u;
	return APO_OK;
}

// After apo_dims_upload / apo_dims_generate: the Form Q (or Form W, below) copy of the engine's fp32 tensor, which resident
// Form D calls read through K1q (route_twin) at 14 (8) instead of 36 bytes per evaluation.  Built when the evaluations are categorical and at least
// kTwinHeadroom of device memory stays free beside it; otherwise Form D is kept alone, without an error.
constexpr uint64_t kTwinHeadroom = 4ull << 30;
int build_twin_wq(apo_engine *e) {
	const uint32_t C = e->dims_C;
	const uint64_t T = e->dims_T, pitch = e->dims_pitch, n = (uint64_t)C * pitch;
	if (e->env_no_twin || C == 0 || T == 0) return APO_OK;
	size_t free_bytes = 0, total_bytes = 0;
	CK(cudaMemGetInfo(&free_bytes, &total_bytes));
	if ((uint64_t)free_bytes < n * 14 + kTwinHeadroom) return APO_OK;
	if (e->q8.reserve(n) != cudaSuccess || e->qd2.reserve(n) != cudaSuccess || e->qli.reserve(n) != cudaSuccess) {
		cudaGetLastError();                                 // another user of the device took the room since cudaMemGetInfo
		e->q8.release(); e->qd2.release(); e->qli.release();
		return APO_OK;
	}
	int rc = compact_begin(e, C, pitch);
	if (rc) return rc;
	CK(apo::run_transcode(e->dims_ptr, pitch, C, T, e->q8.p, e->qd2.p, pitch, e->qbook.p, e->qbook.p + 8 * 256, e->stream));
	rc = compact_finish(e, C, T, pitch, true);
	if (rc != APO_OK) return rc == APO_E_STATE ? APO_OK : rc;
	// A copy whose coded dimensions take at most 15 values each (dense codes 0-14, so 15 can mean absent; true for every tensor
	// TCS:668-763 produces) is kept as Form W words instead: 8 instead of 14 bytes per evaluation.  They are packed from the
	// planes, so the build peaks at the fp32 tensor + the planes + the words; without kTwinHeadroom beside that, Form Q stays.
	for (int j = 0; j < 8; j++)
		if (e->qt.book[256 * j + 15] != 0xFFFFFFFFu) return APO_OK;
	CK(cudaMemGetInfo(&free_bytes, &total_bytes));
	if ((uint64_t)free_bytes < n * 8 + kTwinHeadroom) return APO_OK;
	if (e->qw.reserve(n) != cudaSuccess) { cudaGetLastError(); return APO_OK; }
	CK(apo::run_pack_w(e->q8.p, e->qd2.p, e->qli.p, n, e->qw.p, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	e->q8.release(); e->qd2.release(); e->qli.release();
	e->twin_w = true;
	return APO_OK;
}

int build_twin_t(apo_engine *e);   // beside apo_dims_tuples, whose machinery it uses

// the copies of the engine's freshly loaded fp32 tensor: Form W / Q, then (large tensors) Form T beside it
int build_twin(apo_engine *e) {
	const int rc = build_twin_wq(e);
	return rc == APO_OK && e->twin ? build_twin_t(e) : rc;
}

// true when the driver does not know the pointer: ordinary pageable host memory (malloc, JS ArrayBuffer, numpy)
bool is_pageable(const void *p) {
	cudaPointerAttributes a;
	if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return true; }
	return a.type == cudaMemoryTypeUnregistered;
}

// rows x width bytes, strided -> strided, split over a few host threads (a single memcpy stream does not fill PCIe 5)
void parallel_rows_copy(uint8_t *dst, size_t dpitch, const uint8_t *src, size_t spitch, size_t width, uint32_t rows) {
	unsigned nt = std::thread::hardware_concurrency();
	static const int env_threads = [] { const char *v = getenv("APO_HOST_THREADS"); return v ? atoi(v) : 0; }();   // read once per process
	if (env_threads > 0) nt = (unsigned)env_threads;
	else nt = nt ? (nt > 16 ? 16 : nt) : 4;        // default: at most 16; APO_HOST_THREADS overrides
	if (nt > 64) nt = 64;
	const size_t total = width * rows;
	if (nt == 1 || total < (8u << 20)) { for (uint32_t r = 0; r < rows; r++) memcpy(dst + r * dpitch, src + r * spitch, width); return; }
	// split every row into nt column slices: works for C = 1 as well as for many short rows
	auto work = [&](unsigned k) {
		const size_t lo = width * k / nt, hi = width * (k + 1) / nt;
		for (uint32_t r = 0; r < rows; r++) memcpy(dst + r * dpitch + lo, src + r * spitch + lo, hi - lo);
	};
	std::vector<std::thread> th;
	unsigned started = 1;
	try {
		for (unsigned k = 1; k < nt; k++, started++) th.emplace_back(work, k);
	} catch (...) {}                                   // thread limit reached: the slices not handed out are copied here
	work(0);
	for (unsigned k = started; k < nt; k++) work(k);
	for (auto &t : th) t.join();
}

// two page-locked staging buffers of at least `bytes` each (kept for the life of the handle)
int ensure_stage(apo_engine *e, uint64_t bytes) {
	if (e->h_stage_cap >= bytes) return APO_OK;
	for (int i = 0; i < 2; i++) { if (e->h_stage[i]) cudaFreeHost(e->h_stage[i]); e->h_stage[i] = nullptr; }
	e->h_stage_cap = 0;
	for (int i = 0; i < 2; i++) CK(cudaMallocHost((void **)&e->h_stage[i], bytes));
	e->h_stage_cap = bytes;
	return APO_OK;
}

// cudaMemcpy2DAsync rejects pitches above cudaDeviceProp::memPitch (read at apo_create): rows of a host tensor whose
// record axis is longer than that (T * row bytes > 2 GiB, the "larger than device memory" case of the streaming calls)
// are copied one by one instead.
int copy_rows_h2d(apo_engine *e, void *dst, size_t dpitch, const void *src, size_t spitch, size_t width, uint32_t rows, cudaStream_t st) {
	if (rows == 0 || width == 0) return APO_OK;
	if (rows == 1) { CK(cudaMemcpyAsync(dst, src, width, cudaMemcpyHostToDevice, st)); return APO_OK; }
	if (e->mem_pitch_max == 0 || (dpitch <= e->mem_pitch_max && spitch <= e->mem_pitch_max)) {
		CK(cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, rows, cudaMemcpyHostToDevice, st));
		return APO_OK;
	}
	for (uint32_t r = 0; r < rows; r++)
		CK(cudaMemcpyAsync((uint8_t *)dst + (size_t)r * dpitch, (const uint8_t *)src + (size_t)r * spitch, width, cudaMemcpyHostToDevice, st));
	return APO_OK;
}

// rows x width bytes host -> device on `st` (asynchronous for page-locked sources; a pageable source is fully consumed
// when this returns).  Large pageable sources go through the staging buffers in column slices of all rows.
int h2d_rows(apo_engine *e, void *dst, size_t dpitch, const void *src, size_t spitch, size_t width, uint32_t rows, cudaStream_t st) {
	const uint64_t total = (uint64_t)width * rows;
	if (total < (64ull << 20) || !is_pageable(src) || e->env_no_staging)
		return copy_rows_h2d(e, dst, dpitch, src, spitch, width, rows, st);
	const uint64_t cap = 256ull << 20;
	int rc = ensure_stage(e, cap);
	if (rc) return rc;
	size_t W = (size_t)(cap / rows) & ~(size_t)255;            // slice width per row, 256-byte granular
	if (W == 0) W = 256;
	int k = 0;
	for (size_t w0 = 0; w0 < width; w0 += W, k++) {
		const int b = k & 1;
		const size_t w = width - w0 < W ? width - w0 : W;
		if (k >= 2) CK(cudaEventSynchronize(e->stage_done[b]));
		parallel_rows_copy(e->h_stage[b], W, (const uint8_t *)src + w0, spitch, w, rows);
		{ const int rc2 = copy_rows_h2d(e, (uint8_t *)dst + w0, dpitch, e->h_stage[b], W, w, rows, st); if (rc2) return rc2; }
		CK(cudaEventRecord(e->stage_done[b], st));
	}
	return APO_OK;
}

struct ResultLayout { uint64_t off_scores, off_counts, off_topk, off_report, off_meta, bytes; };
ResultLayout result_layout(uint32_t C, uint32_t K) {
	ResultLayout L;
	L.off_scores = 0;
	L.off_counts = L.off_scores + 8ull * C;
	L.off_topk = L.off_counts + 8ull * C;
	L.off_report = round_up(L.off_topk + 4ull * K, 16);
	L.off_meta = round_up(L.off_report + sizeof(apo_corpus_report), 16);
	L.bytes = L.off_meta + sizeof(apo::ResultMeta);
	return L;
}
static_assert(sizeof(apo::ResultMeta) == 32, "result block stays a multiple of 16 bytes");
constexpr uint64_t kHostOutMax = 64ull << 10;      // result blocks up to this size are written to the caller's page-locked buffer by the kernel itself
constexpr uint64_t kTimingMinBytes = 64ull << 20;  // per-stage CUDA events are recorded for calls streaming at least this much (or on request)
constexpr uint64_t ARM_WORDS = 19;                  // 18 example slots + ticket, right behind the partial vector

int ensure_scratch(apo_engine *e, uint32_t C, uint32_t K) {
	if (acc_words(C, e->nranks) + ARM_WORDS > e->acc.cap) e->acc_clean_words = 0;      // a fresh allocation is not zeroed
	CK(reserve(e, e->acc, acc_words(C, e->nranks) + ARM_WORDS));
	CK(reserve(e, e->acc_snapshot, (uint64_t)ACC_PER_CAND * (C ? C : 1)));
	const ResultLayout L = result_layout(C, K);
	CK(reserve(e, e->result, L.bytes));
	CK(reserve(e, e->keys, C ? C : 1));
	CK(reserve(e, e->sel_key, K ? K : 1));
	CK(reserve(e, e->sel_idx, K ? K : 1));
	if (e->nranks > 1) CK(reserve(e, e->acc_joined, acc_words(C, e->nranks)));
	if (e->h_result_cap < L.bytes) {
		if (e->h_result) cudaFreeHost(e->h_result);
		e->h_result = nullptr; e->h_result_cap = 0;
		CK(cudaMallocHost((void **)&e->h_result, L.bytes));
		e->h_result_cap = L.bytes;
	}
	return APO_OK;
}

// the peer-memory join is used when the block exists on every rank and the partial vector fits its slots
bool peer_join_active(const apo_engine *e, uint32_t C) {
	return e->nranks > 1 && e->peer_ok && !e->env_nccl_join && acc_words(C, e->nranks) <= e->peer_slot_words;
}

// layout of one rank's peer block: [PEER_MAX] arrival flags | [PEER_MAX] done-reading flags (128 B) | slot 0 | slot 1
constexpr uint64_t kPeerHeader = 2 * apo::PEER_MAX * 8;
inline unsigned long long *peer_flags(void *base) { return (unsigned long long *)base; }
inline long long *peer_slot(void *base, uint64_t slot_words, int parity) { return (long long *)((uint8_t *)base + kPeerHeader) + (uint64_t)parity * slot_words; }

apo::FinalizeParams make_fin(apo_engine *e, uint32_t C, uint32_t K, int with_corpus) {
	const ResultLayout L = result_layout(C, K);
	apo::FinalizeParams F{};
	F.acc = e->acc.p; F.C = C; F.K = K; F.nranks = e->nranks; F.with_corpus = with_corpus;
	F.scores = (double *)(e->result.p + L.off_scores);
	F.counts = (uint64_t *)(e->result.p + L.off_counts);
	F.keys = e->keys.p; F.sel_key = e->sel_key.p; F.sel_idx = e->sel_idx.p;
	F.topk = (int32_t *)(e->result.p + L.off_topk);
	F.report = (apo_corpus_report *)(e->result.p + L.off_report);
	F.result_base = e->result.p; F.result_bytes = (uint32_t)L.bytes; F.meta_off = (uint32_t)L.off_meta;
	F.host_out = L.bytes <= kHostOutMax ? e->h_result : nullptr;
	F.join.nranks = 1;
	if (peer_join_active(e, C)) {
		apo::JoinParams &J = F.join;
		J.nranks = e->nranks; J.rank = e->rank; J.words = (uint32_t)acc_words(C, e->nranks); J.epoch = e->join_epoch;
		for (int r = 0; r < e->nranks; r++) {
			J.slot[r] = peer_slot(e->peer_base[r], e->peer_slot_words, (int)(e->join_epoch & 1ull));
			J.flag[r] = peer_flags(e->peer_base[r]);
		}
		J.joined = e->acc_joined.p;
	}
	return F;
}

// zero the candidate accumulators of a scoring session
int begin_score(apo_engine *e, uint32_t C, bool whole = false) {
	// whole: also the corpus block, the example scratch and the ticket (one-shot calls: a single memset arms everything —
	// and none at all when the previous one-shot call left the block zeroed, see FinalizeParams::clean_ptr)
	const uint64_t words = whole ? acc_words(C, e->nranks) + ARM_WORDS : (uint64_t)ACC_PER_CAND * C;
	if (!(whole && e->acc_clean_words >= words)) CK(cudaMemsetAsync(e->acc.p, 0, words * 8, e->stream));
	e->acc_clean_words = 0;                         // from here on the block is in use
	*e->h_domain = 0u;                              // the previous call has been synchronised: no kernel writes it now
	e->partials_src = e->nranks > 1 ? e->acc_joined.p : e->acc.p;
	e->last_C = C; e->score_C = C; e->scoring = true; e->k1_used = 0;
	e->cand_armed = false; e->cand_every = true; e->cand_ready = false;
	e->ccorp_armed = false; e->ccorp_every = true; e->ccorp_ready = false;
	e->timing = apo_timing{};
	if (e->timing_on) CK(cudaEventRecord(e->ev[0], e->stream));
	return APO_OK;
}

int record_k1_event(apo_engine *e, int which) {
	if (!e->timing_on) return APO_OK;
	if (which == 0 && e->k1_used + 2 > e->k1_ev.size()) {
		for (int i = 0; i < 2; i++) { cudaEvent_t ev; CK(cudaEventCreate(&ev)); e->k1_ev.push_back(ev); }
	}
	CK(cudaEventRecord(e->k1_ev[e->k1_used + which], e->stream));
	if (which == 1) e->k1_used += 2;
	return APO_OK;
}

// Form T: the table values of every entry of d for the current weights and `recip` into v (k_tuple_values).  Held values
// (the copy): into the buffers build_twin_t allocated, so a scoring call allocates nothing after route_twin; then waits and
// records whether every entry lies in Form T's domain.  Otherwise device work on e->stream only, which the call checks once
// it has synchronised (finish_score).
int tuple_values(apo_engine *e, const TupleDict &d, TupleVals &v, bool recip) {
	const std::vector<double> tab = make_ptab(d.book, e->W, std::nan(""));
	if (!v.held) {
		CK(reserve(e, v.ptab, 8 * 256));
		CK(reserve(e, v.val[0], (uint64_t)d.n + 1));
		CK(reserve(e, v.bad, 1));
	}
	CK(cudaMemcpyAsync(v.ptab.p, tab.data(), 8 * 256 * 8, cudaMemcpyHostToDevice, e->stream));   // pageable source: consumed when this returns
	if (e->tvals_check != &v) CK(cudaMemsetAsync(v.bad.p, 0, 4, e->stream));   // a session keeps the flags of its earlier launches
	apo::TupleValParams V{};
	V.tb_pc = d.pc.p; V.tb_pd = d.pd.p; V.n = d.n; V.ptab = v.ptab.p; V.lut = e->d_lut.p; V.d2book = d.d2.p; V.w2 = e->W.w[2];
	V.tval = v.out(recip); V.bad = v.bad.p;
	CK(apo::run_tuple_values(V, recip, e->stream));
	if (!v.held) { e->timing.launches++; e->tvals_check = &v; return APO_OK; }
	uint32_t bad = 0;
	CK(cudaMemcpyAsync(&bad, v.bad.p, 4, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	v.ok[recip] = bad ? 2 : 1;
	return APO_OK;
}

// a resident Form D call: the copy's values for its `recip`, computed once per weight set by the first call that needs them
int twin_t_ready(apo_engine *e, const apo_score_opts *o) {
	const bool recip = (o->flags & APO_SCORE_RECIP) != 0;
	if (o->source != APO_SRC_DIMS || e->tcopy.C == 0 || e->env_no_twin_t || e->tcopy.vals.ok[recip]) return APO_OK;
	return tuple_values(e, e->tcopy, e->tcopy.vals, recip);
}

// ---- the evaluations one launch reads: a resident tensor (or a window of it), or one window of a host-streaming call
using Form = apo::CandSource;   // the five layouts: CAND_DIMS (Form D), CAND_REC32 / CAND_REC16 (Form R / R16), CAND_Q, CAND_T

struct Evals {
	Form form = apo::CAND_DIMS;
	int variant = 0;                          // kernel variant (Form Q: after the fall-back to the product tables)
	uint32_t C = 0;
	uint64_t count = 0;                       // evaluations per candidate
	uint64_t pitch_evals = 0;                 // candidate row pitch
	uint64_t idx_base = 0;                    // record position of evaluation 0: the window start or the streamed chunk start
	const uint8_t *rows = nullptr;            // Form D / R / R16: evaluation 0 of candidate 0
	const unsigned long long *q8 = nullptr;   // Form Q planes
	const float *d2 = nullptr;
	const unsigned short *li = nullptr;
	const QTables *qt = nullptr;              // Form Q / W: K1q's tables of the codebook
	const unsigned long long *qw = nullptr;   // Form W words (the copy of a resident Form D tensor, route_twin)
	const unsigned short *tl = nullptr;       // Form T planes
	const unsigned char *th = nullptr;
	const TupleDict *dict = nullptr;          // Form T dictionary and its values: held (the copy, route_twin), computed by every
	TupleVals *tv = nullptr;                  // launch (resident Form T) or, t_once, once for the whole call together with the
	bool t_once = false;                      // breakdown's codebook table (host streaming)
	bool t2 = false;                          // the Form T copy through K1t2: tl and the exception list, not th (route_twin)

	bool records() const { return form == apo::CAND_REC32 || form == apo::CAND_REC16; }
	uint32_t row() const { return form == apo::CAND_DIMS ? 36 : form == apo::CAND_REC32 ? 32 : 16; }
	uint32_t bytes() const { return form == apo::CAND_T ? (t2 ? 2 : 3) : form == apo::CAND_Q ? 14 : form == apo::CAND_W ? 8 : row(); }   // read per evaluation
	uint64_t tile() const {                   // evaluations per tile of the scoring kernel
		return (uint64_t)(form == apo::CAND_T ? (t2 ? apo::kt2_tile_evals() : apo::kt_tile_evals()) : form == apo::CAND_Q ? apo::kq_tile_evals(variant)
		                  : form == apo::CAND_W ? apo::kw_tile_evals() : apo::k1_tile_evals((int)row(), variant));
	}
};

// ev reads all of the resident Form T tensor t with the values v
void resident_tuples(Evals *ev, const TupleTensor &t, TupleVals &v) {
	ev->form = apo::CAND_T; ev->C = t.C; ev->count = t.T; ev->pitch_evals = t.pitch;
	ev->tl = t.l.p; ev->th = t.h.p; ev->dict = &t; ev->tv = &v;
}

// the whole tensor loaded for o->source (count = all its evaluations)
int resident_evals(apo_engine *e, const apo_score_opts *o, Evals *ev) {
	if (!o) return fail(e, APO_E_ARG, "opts is NULL");
	if (o->source > APO_SRC_TUPLES) return fail(e, APO_E_ARG, "unknown source %u", o->source);
	Evals &v = *ev;
	v = Evals{};
	v.variant = (int)o->variant;
	if (o->source == APO_SRC_TUPLES) {
		if (e->tup.l.p == nullptr || e->tup.C == 0) return fail(e, APO_E_STATE, "no tuples loaded");
		resident_tuples(&v, e->tup, e->tvals);
	} else if (o->source == APO_SRC_ROLLOUTS) {
		if (e->roll.p == nullptr || e->roll_C == 0) return fail(e, APO_E_STATE, "no rollouts loaded");
		v.form = e->roll_row == 32 ? apo::CAND_REC32 : apo::CAND_REC16; v.C = e->roll_C; v.count = e->roll_T; v.pitch_evals = e->roll_pitch;
		v.rows = e->roll.p;
	} else {
		if ((e->dims_ptr == nullptr && !e->compact) || e->dims_C == 0) return fail(e, APO_E_STATE, "no dims loaded");
		v.C = e->dims_C; v.count = e->dims_T; v.pitch_evals = e->dims_pitch;
		if (e->compact) {
			v.form = apo::CAND_Q; v.q8 = e->q8.p; v.d2 = e->qd2.p; v.li = e->qli.p; v.qt = &e->qt;
			if ((v.variant == 0 || v.variant >= 5) && !e->qt.pair_ok) v.variant = 4;   // prefix table would not fit: product tables only
		} else {
			v.rows = (const uint8_t *)e->dims_ptr;
		}
	}
	return APO_OK;
}

// ev narrowed to o's window, which check_window has placed inside it
int resident_window(apo_engine *e, const apo_score_opts *o, Evals *ev) {
	const uint64_t first = o->first;
	ev->count = o->count ? o->count : ev->count - first;
	if (ev->count && first % 8 && ev->form == apo::CAND_T) return fail(e, APO_E_ARG, "window start must be a multiple of 8 for Form T");
	if (ev->count && first % 8 && ev->form == apo::CAND_Q) return fail(e, APO_E_ARG, "window start must be a multiple of 8 for the compact layout");
	ev->idx_base = first;
	if (ev->rows) ev->rows += first * ev->row();
	if (ev->q8) { ev->q8 += first; ev->d2 += first; ev->li += first; }
	if (ev->qw) ev->qw += first;
	if (ev->tl) { ev->tl += first; ev->th += first; }
	return APO_OK;
}

// A resident Form D call reads the Form Q / W copy through K1q instead when one is held, the variant is the default (1-4 name
// K1 tile shapes) and the window starts on K1q's 8-evaluation grid; under the same conditions it reads the Form T copy through
// K1t when that is held and its values for this call's weights and `recip` are valid (twin_t_ready): through K1t2 from the
// 16-bit plane when the copy holds an exception list and APO_TUNE_NO_TWIN_T2 is clear.  Before resident_window, after the
// call's last allocation before its launches (reserve may release the copies).
void route_twin(apo_engine *e, const apo_score_opts *o, Evals *ev) {
	if (ev->form != apo::CAND_DIMS || !e->twin || e->env_no_twin || o->variant != 0 || o->first % 8) return;
	ev->rows = nullptr;
	if (e->tcopy.C && !e->env_no_twin_t && e->tcopy.vals.ok[(o->flags & APO_SCORE_RECIP) != 0] == 1) {
		resident_tuples(ev, e->tcopy, e->tcopy.vals);
		ev->variant = 0;
		ev->t2 = e->tcopy.t2 && !e->env_no_twin_t2;
		return;
	}
	ev->qt = &e->qt;
	if (e->twin_w) {                                         // <= 15 codes per dimension: the prefix table always fits
		ev->form = apo::CAND_W; ev->qw = e->qw.p; ev->variant = 0;
		return;
	}
	ev->form = apo::CAND_Q;
	ev->q8 = e->q8.p; ev->d2 = e->qd2.p; ev->li = e->qli.p;
	ev->variant = e->qt.pair_ok ? 0 : 4;                     // as resident_evals for a compact tensor
}

// one scoring launch (K1 / K1q / K1t) over ev into candidates [cand_offset, ...); fused: the corpus scan and the tail ride on it
int launch_score(apo_engine *e, const apo_score_opts *o, const Evals &ev, uint32_t cand_offset, const apo::K2Params *fused = nullptr) {
	if (!ev.count) return APO_OK;
	const bool recip = (o->flags & APO_SCORE_RECIP) != 0;
	long long *acc = e->acc.p + (uint64_t)ACC_PER_CAND * cand_offset;
	int rc;
	if (ev.form == apo::CAND_T && !ev.t_once && !ev.tv->held && (rc = tuple_values(e, *ev.dict, *ev.tv, recip))) return rc;
	if ((rc = record_k1_event(e, 0))) return rc;
	if (ev.form == apo::CAND_T && ev.t2) {
		apo::Kt2Params P{};
		P.tl = ev.tl; P.pitch_evals = ev.pitch_evals; P.C = ev.C; P.T = ev.count; P.first = ev.idx_base;
		P.acc = acc; P.tval = ev.tv->out(recip); P.n_tuples = ev.dict->n;
		P.xs = e->tcopy.xs.p; P.xb = e->tcopy.xb.p; P.xb_pitch = e->tcopy.nblk + 1;   // only the copy holds an exception list
		CK(apo::run_reward9t2(P, e->sm_count, e->stream));
	} else if (ev.form == apo::CAND_T) {
		apo::KtParams P{};
		P.tl = ev.tl; P.th = ev.th; P.pitch_evals = ev.pitch_evals; P.C = ev.C; P.T = ev.count;
		P.acc = acc; P.n_tuples = ev.dict->n; P.tval = ev.tv->out(recip); P.bad = ev.tv->bad.p;
		CK(apo::run_reward9t(P, e->sm_count, e->stream));
	} else if (ev.form == apo::CAND_Q || ev.form == apo::CAND_W) {
		apo::KqParams Q{};
		Q.q8 = ev.q8; Q.d2 = ev.d2; Q.li = ev.li; Q.qw = ev.qw; Q.pitch_evals = ev.pitch_evals; Q.C = ev.C; Q.T = ev.count;
		Q.acc = acc; Q.lut = e->d_lut.p; Q.ptab = ev.qt->ptab.p; Q.w2 = e->W.w[2];
		Q.pair = ev.qt->pair.p; Q.cbf = ev.qt->cbf.p; Q.n0 = ev.qt->n0; Q.n1 = ev.qt->n1;
		for (int j = 0; j < 8; j++) Q.wq[j] = e->W.w[kCodedDim[j]];
		Q.bad = (uint32_t *)e->h_domain;
		if (fused) { Q.corpus_on = 1; Q.corpus = *fused; }
		CK(apo::run_reward9q(Q, ev.variant, recip, e->sm_count, e->stream));
	} else {
		apo::K1Params P{};
		P.base = ev.rows; P.pitch_bytes = ev.pitch_evals * ev.row(); P.C = ev.C; P.T = ev.count; P.acc = acc;
		P.lut = e->d_lut.p;
		P.W = e->W;
		P.bad = (uint32_t *)e->h_domain;
		if (fused) { P.corpus_on = 1; P.corpus = *fused; }
		CK(apo::run_reward9(P, (int)ev.row(), ev.variant, recip, e->sm_count, e->stream));
	}
	if ((rc = record_k1_event(e, 1))) return rc;
	e->timing.launches++;
	return APO_OK;
}

// ---- per-candidate breakdown (APO_SCORE_CANDIDATES)
bool wants_cand(const apo_score_opts *o) { return (o->flags & APO_SCORE_CANDIDATES) != 0; }

int cand_check(apo_engine *e) {
	if (e->nranks > 1)
		return fail(e, APO_E_STATE, "APO_SCORE_CANDIDATES is single-rank only: the per-candidate breakdown is not joined across the %d ranks of this handle", e->nranks);
	return APO_OK;
}

// the breakdown's buffers (cand_arm's, and cand_upload_tbook's for Form T), allocated before route_twin
uint64_t cand_words(uint32_t C) { return (uint64_t)C * (apo::CB_INT + 3) + 1; }

int cand_reserve(apo_engine *e, uint32_t C) {
	CK(reserve(e, e->cand_acc, cand_words(C)));
	CK(reserve(e, e->cand_book, 8 * 16));
	return APO_OK;
}

// zero the breakdown of C candidates (first flagged launch of a call or session)
int cand_arm(apo_engine *e, uint32_t C) {
	const uint64_t words = cand_words(C);
	CK(reserve(e, e->cand_acc, words));
	CK(cudaMemsetAsync(e->cand_acc.p, 0, words * 8, e->stream));
	e->cand_armed = true;
	return APO_OK;
}

// Form T dictionary codebook -> [8][16] fp32 values (4-bit codes, csrc/apo_tuple.cu)
int cand_upload_tbook(apo_engine *e, const uint32_t *codebook) {
	uint32_t tab[8 * 16];
	for (int j = 0; j < 8; j++) for (int k = 0; k < 16; k++) tab[16 * j + k] = codebook[256 * j + k];
	CK(reserve(e, e->cand_book, 8 * 16));
	CK(cudaMemcpyAsync(e->cand_book.p, tab, sizeof tab, cudaMemcpyHostToDevice, e->stream));   // pageable source: consumed when this returns
	return APO_OK;
}

// the breakdown pass over ev into candidates [cand_offset, ...)
int launch_cand(apo_engine *e, const Evals &ev, uint32_t cand_offset) {
	if (!ev.count) return APO_OK;
	if (ev.form == apo::CAND_T && !ev.t_once) { const int rc = cand_upload_tbook(e, ev.dict->book); if (rc) return rc; }
	apo::CandParams P{};
	P.C = ev.C; P.T = ev.count; P.idx_base = ev.idx_base; P.pitch_evals = ev.pitch_evals; P.lut = e->d_lut.p;
	P.ints = e->cand_acc.p + (uint64_t)apo::CB_INT * cand_offset;
	P.ex = (unsigned long long *)(e->cand_acc.p + (uint64_t)apo::CB_INT * e->score_C) + 3ull * cand_offset;
	P.dom = (unsigned int *)(e->cand_acc.p + cand_words(e->score_C) - 1);
	P.rows = ev.rows; P.q8 = ev.q8; P.d2 = ev.d2; P.li = ev.li; P.qw = ev.qw;
	P.tl = ev.tl; P.th = ev.th;
	if (ev.qt) P.cbf = ev.qt->cbf.p;
	if (ev.form == apo::CAND_T) {
		P.tb_pc = ev.dict->pc.p; P.tb_pd = ev.dict->pd.p; P.n_tuples = ev.dict->n; P.d2book = ev.dict->d2.p; P.tbook = e->cand_book.p;
	}
	CK(apo::run_cand_breakdown(P, ev.form, e->sm_count, e->stream));
	e->timing.launches++;
	return APO_OK;
}

// integers -> apo_candidate_report[C]; after the scoring call has completed (its partials are final)
int cand_finish(apo_engine *e, uint32_t C) {
	CK(reserve(e, e->cand_rep, C ? C : 1));
	const long long *partials = e->partials_src ? e->partials_src : e->acc.p;
	CK(apo::run_cand_report(e->cand_acc.p, (const unsigned long long *)(e->cand_acc.p + (uint64_t)apo::CB_INT * C), partials, C, e->cand_rep.p, e->stream));
	e->timing.launches++;
	uint32_t dom = 0;                                              // k_cand_breakdown's domain word (pageable: the copy waits for the stream)
	CK(cudaMemcpyAsync(&dom, e->cand_acc.p + cand_words(C) - 1, 4, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	if (dom)
		return fail(e, APO_E_ARG, "APO_SCORE_CANDIDATES: an evaluation with a finalReward has a dimension with |v| >= 2048 (or NaN), "
		                          "whose rint(v * 2^52) has no exact fixed-point sum");
	e->cand_C = C; e->cand_ready = true;
	return APO_OK;
}

// ---- per-candidate corpus report (APO_SCORE_CANDIDATE_CORPUS)
bool wants_ccorp(const apo_score_opts *o) { return (o->flags & APO_SCORE_CANDIDATE_CORPUS) != 0; }

// records: the call reads trace records (Form R / R16); the other forms carry only the nine reward values
int ccorp_check(apo_engine *e, bool records) {
	if (!records)
		return fail(e, APO_E_ARG, "APO_SCORE_CANDIDATE_CORPUS needs rollout records (Form R / R16): this source holds reward values only, "
		                          "without the fields the patterns, modes and tool totals read");
	if (e->nranks > 1)
		return fail(e, APO_E_STATE, "APO_SCORE_CANDIDATE_CORPUS is single-rank only: the per-candidate corpus reports are not joined across the %d ranks of this handle", e->nranks);
	return APO_OK;
}

// zero the corpus blocks of C candidates (first flagged launch of a call or session)
int ccorp_arm(apo_engine *e, uint32_t C) {
	const uint64_t words = (uint64_t)C * apo::CC_WORDS;
	CK(reserve(e, e->ccorp_acc, 2 * words));                 // blocks | report scratch
	CK(cudaMemsetAsync(e->ccorp_acc.p, 0, words * 8, e->stream));
	e->ccorp_armed = true;
	return APO_OK;
}

// corpus scan of ev's trace records (Form R / R16) into candidates [cand_offset, ...)
int launch_ccorp(apo_engine *e, const Evals &ev, uint32_t cand_offset) {
	if (!ev.count) return APO_OK;
	apo::CandCorpusParams P{};
	P.C = ev.C; P.T = ev.count; P.idx_base = ev.idx_base; P.pitch_evals = ev.pitch_evals; P.rows = ev.rows;
	P.lut = e->d_lut.p; P.w2 = e->W.w[2];
	P.blk = e->ccorp_acc.p + (uint64_t)apo::CC_WORDS * cand_offset;
	CK(apo::run_cand_corpus(P, (int)ev.row(), e->sm_count, e->stream));
	e->timing.launches++;
	return APO_OK;
}

// blocks -> apo_corpus_report[C]
int ccorp_finish(apo_engine *e, uint32_t C) {
	CK(reserve(e, e->ccorp_rep, C ? C : 1));
	CK(apo::run_cand_corpus_report(e->ccorp_acc.p, C, e->ccorp_rep.p, e->stream));
	e->timing.launches++;
	CK(cudaStreamSynchronize(e->stream));
	e->ccorp_C = C; e->ccorp_ready = true;
	return APO_OK;
}

// K2 (+fused finalize) / allreduce / K3, then bring the result block home
bool wants_corpus(const apo_engine *e, const apo_score_opts *o) { return (o->flags & APO_SCORE_CORPUS) && e->corpus_T > 0; }

// the corpus block, the example scratch and the ticket belong to one corpus pass only, so that a scoring session can be
// finished repeatedly while evaluations keep being accumulated (incremental scoring); they sit behind the candidate
// accumulators in one allocation: one memset
int arm_corpus(apo_engine *e, uint32_t C) {
	CK(cudaMemsetAsync(e->acc.p + (uint64_t)ACC_PER_CAND * C, 0, (CORP_FIXED + 18ull * e->nranks + ARM_WORDS) * 8, e->stream));
	return APO_OK;
}

apo::K2Params make_k2(apo_engine *e, uint32_t C, const apo::FinalizeParams &F) {
	apo::K2Params P{};
	unsigned long long *arm = (unsigned long long *)(e->acc.p + acc_words(C, e->nranks));
	P.recs = e->corpus.p; P.T = e->corpus_T; P.idx_base = e->corpus_base; P.C = C; P.rank = e->rank;
	P.acc = e->acc.p; P.ex_scratch = arm; P.ticket = (unsigned int *)(arm + 18);
	P.lut = e->d_lut.p; P.W = e->W; P.fuse_finalize = (e->nranks == 1 || F.join.nranks > 1) ? 1 : 0; P.fin = F;
	return P;
}

// The end of every scoring call: the result, then the per-candidate reports it asked for.  fused_corpus: the scoring kernel
// already ran the corpus scan; at one rank or with the peer join its last CTA also finalised and left the accumulator block
// zeroed (apo_score sets FinalizeParams::clean_ptr).  unpacked: Form P, whose k_unpack_p flags evaluations naming empty slots.
int finish_score(apo_engine *e, const apo_score_opts *o, uint32_t C, double *scores, uint64_t *counts, int32_t *topk,
                 apo_corpus_report *report, bool fused_corpus = false, bool unpacked = false) {
	const uint32_t K = o->K;
	const bool with_corpus = wants_corpus(e, o);
	const bool tm = e->timing_on;
	apo::FinalizeParams F = make_fin(e, C, K, with_corpus ? 1 : 0);
	const bool peer = F.join.nranks > 1;
	int rc;
	if (!fused_corpus && (rc = arm_corpus(e, C))) return rc;
	if (tm) CK(cudaEventRecord(e->ev[1], e->stream));
	const bool self_clean = fused_corpus && (e->nranks == 1 || peer);
	bool finalized = self_clean;
	if (with_corpus && !fused_corpus) {
		const apo::K2Params P = make_k2(e, C, F);
		CK(apo::run_detect6(P, e->sm_count, e->stream));
		e->timing.launches++;
		finalized = P.fuse_finalize != 0;
	}
	if (tm) CK(cudaEventRecord(e->ev[2], e->stream));
	if (e->nranks > 1 && !peer) {
		const int rc = g_nccl.AllReduce(e->acc.p, e->acc_joined.p, (size_t)acc_words(C, e->nranks), kNcclInt64, kNcclSum, e->comm, e->stream);
		if (rc != 0) return fail(e, APO_E_NCCL, "ncclAllReduce: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "error");
		e->timing.launches++;
		F.acc = e->acc_joined.p;
	}
	if (tm) CK(cudaEventRecord(e->ev[3], e->stream));
	if (!finalized) {
		CK(apo::run_finalize(F, e->stream));
		e->timing.launches++;
	}
	if (tm) CK(cudaEventRecord(e->ev[4], e->stream));
	const ResultLayout L = result_layout(C, K);
	if (!F.host_out) CK(cudaMemcpyAsync(e->h_result, e->result.p, L.bytes, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	apo::ResultMeta meta;
	memcpy(&meta, e->h_result + L.off_meta, sizeof meta);
	if (meta.status != 0)
		return fail(e, APO_E_NCCL, "peer-memory join timed out after %.0f ms: a rank did not reach the join of call %llu", meta.join_wait_us * 1e-3,
		            (unsigned long long)e->join_epoch);
	if (*e->h_domain)
		return fail(e, APO_E_ARG, "an evaluation's finalReward is outside [-512, 512) (a dimension beyond +-512, +-inf): outside the exact fixed-point domain");
	if (self_clean) {
		e->acc_clean_words = acc_words(C, e->nranks) + ARM_WORDS;
		if (e->nranks == 1) e->partials_src = e->acc_snapshot.p;
	}
	if (scores) memcpy(scores, e->h_result + L.off_scores, 8ull * C);
	if (counts) memcpy(counts, e->h_result + L.off_counts, 8ull * C);
	if (topk && K) memcpy(topk, e->h_result + L.off_topk, 4ull * (K < C ? K : C));
	if (report) {
		if (with_corpus) memcpy(report, e->h_result + L.off_report, sizeof(apo_corpus_report));
		else memset(report, 0, sizeof(apo_corpus_report));
	}
	e->timing.join_wait_ms = meta.join_wait_us * 1e-3f;
	e->timing.join_reduce_ms = meta.join_reduce_us * 1e-3f;
	e->timing.tail_finalize_ms = meta.finalize_us * 1e-3f;
	e->timing.tail_publish_ms = meta.publish_us * 1e-3f;
	if (tm) {
		float ms = 0;
		e->timing.reward_ms = 0;
		for (size_t i = 0; i + 1 < e->k1_used; i += 2) { cudaEventElapsedTime(&ms, e->k1_ev[i], e->k1_ev[i + 1]); e->timing.reward_ms += ms; }
		cudaEventElapsedTime(&ms, e->ev[1], e->ev[2]); e->timing.corpus_ms = ms;
		cudaEventElapsedTime(&ms, e->ev[2], e->ev[3]); e->timing.allreduce_ms = ms;
		cudaEventElapsedTime(&ms, e->ev[3], e->ev[4]); e->timing.finalize_ms = ms;
		cudaEventElapsedTime(&ms, e->ev[0], e->ev[4]); e->timing.total_ms = ms;
	}
	if (const TupleVals *v = e->tvals_check) {                     // did K1t meet an index outside the dictionary, or an entry it cannot hold?
		e->tvals_check = nullptr;
		uint32_t bad = 0;
		CK(cudaMemcpyAsync(&bad, v->bad.p, 4, cudaMemcpyDeviceToHost, e->stream));
		CK(cudaStreamSynchronize(e->stream));
		if (bad & 2u) return fail(e, APO_E_ARG, "a dictionary entry is not representable in Form T (finalReward outside (-2, 2), or a tool_success_rate index without a value)");
		if (bad & 1u) return fail(e, APO_E_ARG, "a tuple index is outside the dictionary");
	}
	if (unpacked) {                                                // the stream is synchronised
		uint32_t bad = 0;
		CK(cudaMemcpyAsync(&bad, e->unpack_bad.p, 4, cudaMemcpyDeviceToHost, e->stream));
		CK(cudaStreamSynchronize(e->stream));
		if (bad) return fail(e, APO_E_ARG, "an evaluation names an empty or NaN slot of the codebook or of d2book");
	}
	if (wants_cand(o) && (rc = cand_finish(e, C))) return rc;
	return wants_ccorp(o) ? ccorp_finish(e, C) : APO_OK;
}

// o's window against the T evaluations loaded
int check_window(apo_engine *e, const apo_score_opts *o, uint64_t T) {
	if (o->first % 4) return fail(e, APO_E_ARG, "window start must be a multiple of 4");
	if (o->first > T || (o->count && o->first + o->count > T)) return fail(e, APO_E_ARG, "window outside [0,%llu)", (unsigned long long)T);
	return APO_OK;
}

// score_check's T for the host-streaming calls (they take no window) and for apo_score_finish (each accumulate checked its own)
constexpr uint64_t kStreamed = ~0ull, kSession = ~0ull - 1;

// The refusals apo_score, apo_score_finish and the host-streaming calls share, once each has checked its source, in this
// order: beam width, window (inside the T evaluations loaded), per-candidate passes (records: the source holds trace
// records); then the device and the scratch of C candidates.
int score_check(apo_engine *e, const apo_score_opts *o, uint32_t C, uint64_t T, bool records) {
	if (o->K > C) return fail(e, APO_E_ARG, "K=%u exceeds the number of candidates C=%u", o->K, C);
	if (o->K > kMaxK) return fail(e, APO_E_ARG, "K=%u exceeds the supported beam width %u", o->K, kMaxK);
	int rc;
	if (T == kStreamed) {
		if (o->first || o->count) return fail(e, APO_E_ARG, "windows are not supported by the host-streaming calls");
	} else if (T != kSession && (rc = check_window(e, o, T))) {
		return rc;
	}
	if (wants_cand(o) && (rc = cand_check(e))) return rc;
	if (wants_ccorp(o) && (rc = ccorp_check(e, records))) return rc;
	CK(cudaSetDevice(e->device));
	if (T == kSession) return APO_OK;                               // a session's scratch was sized by apo_score_begin
	if ((rc = ensure_scratch(e, C, o->K))) return rc;
	if (wants_cand(o) && (rc = cand_reserve(e, C))) return rc;
	return APO_OK;
}

// The start of the launches: for a new call (begin) the timing choice over `bytes` streamed and the zeroed accumulators (whole:
// a one-shot call's corpus block too, begin_score); then the join epoch, and the per-candidate passes armed unless an
// accumulate of the session has armed them.
int score_arm(apo_engine *e, const apo_score_opts *o, uint32_t C, bool begin, uint64_t bytes = 0, bool whole = false) {
	// per-stage CUDA events cost ~1 us each on the host: record them for calls that stream enough for it not to matter, or on request
	if (begin) e->timing_on = (o->flags & APO_SCORE_TIMING) != 0 || bytes >= kTimingMinBytes;
	if (peer_join_active(e, C)) e->join_epoch++;          // counts joined calls only: consecutive joins alternate between the two export slots
	int rc;
	if (begin && (rc = begin_score(e, C, whole))) return rc;
	if (wants_cand(o) && !e->cand_armed && (rc = cand_arm(e, C))) return rc;
	return wants_ccorp(o) && !e->ccorp_armed ? ccorp_arm(e, C) : APO_OK;
}

}  // namespace

namespace {
struct PeerInfo {                        // exchanged with ncclAllGather at apo_comm_init, 128 bytes per rank
	cudaIpcMemHandle_t handle;           // 64 B
	uint64_t pid, ptr, host_hash;
	int32_t device, ok;
	uint8_t pad[128 - 64 - 24 - 8];
};
static_assert(sizeof(PeerInfo) == 128, "PeerInfo is exchanged as 128 raw bytes");

void peer_teardown(apo_engine *e) {
	if (e->peer_ok && e->peer_block && e->join_epoch > 0) {
		// peers read this block with NVLink loads inside their own launches: wait (bounded) until every peer has signalled
		// that it finished reading the last joined call before the memory goes away
		unsigned long long done[apo::PEER_MAX];
		for (int spin = 0; spin < 2000; spin++) {
			if (cudaMemcpy(done, e->peer_block + apo::PEER_MAX * 8, sizeof done, cudaMemcpyDeviceToHost) != cudaSuccess) { cudaGetLastError(); break; }
			bool all = true;
			for (int r = 0; r < e->nranks; r++) if (r != e->rank && done[r] < e->join_epoch) all = false;
			if (all) break;
			usleep(1000);
		}
	}
	for (int r = 0; r < apo::PEER_MAX; r++) {
		if (e->peer_base[r] && e->peer_ipc[r]) cudaIpcCloseMemHandle(e->peer_base[r]);
		e->peer_base[r] = nullptr; e->peer_ipc[r] = false;
	}
	if (e->peer_block) cudaFree(e->peer_block);
	e->peer_block = nullptr; e->peer_ok = false; e->peer_slot_words = 0;
}

// Allocate this rank's block, exchange handles, map the peers.  Any failure leaves peer_ok false on EVERY rank (the
// outcome is agreed with one ncclAllReduce(min)) and the join falls back to ncclAllReduce + k_finalize.
int peer_setup(apo_engine *e) {
	peer_teardown(e);
	if (e->nranks > apo::PEER_MAX || !g_nccl.AllGather) return APO_OK;
	const uint64_t slot_words = acc_words(16384, e->nranks);          // candidates up to the top-K limit fit a slot (~0.5 MB)
	const uint64_t bytes = kPeerHeader + 2 * slot_words * 8;
	PeerInfo mine{};
	mine.ok = 1;
	if (cudaMalloc((void **)&e->peer_block, bytes) != cudaSuccess) { cudaGetLastError(); e->peer_block = nullptr; mine.ok = 0; }
	if (mine.ok && cudaMemsetAsync(e->peer_block, 0, bytes, e->stream) != cudaSuccess) { cudaGetLastError(); mine.ok = 0; }
	if (mine.ok && cudaIpcGetMemHandle(&mine.handle, e->peer_block) != cudaSuccess) { cudaGetLastError(); mine.ok = 0; }
	mine.pid = (uint64_t)getpid(); mine.ptr = (uint64_t)(uintptr_t)e->peer_block; mine.device = e->device;
	{
		char host[256] = {0};
		gethostname(host, sizeof host - 1);
		uint64_t h = 1469598103934665603ull;
		for (const char *c = host; *c; c++) h = (h ^ (uint8_t)*c) * 1099511628211ull;
		mine.host_hash = h;
	}
	struct Scoped : DevBuf<uint8_t> { ~Scoped() { release(); } } xch;      // freed on every return path
	CK(xch.reserve(128ull * (e->nranks + 1)));
	std::vector<PeerInfo> all(e->nranks);
	CK(cudaMemcpyAsync(xch.p, &mine, 128, cudaMemcpyHostToDevice, e->stream));
	int rc = g_nccl.AllGather(xch.p, xch.p + 128, 128, kNcclInt8, e->comm, e->stream);
	if (rc != 0) { return fail(e, APO_E_NCCL, "ncclAllGather (peer handles): %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "error"); }
	CK(cudaMemcpyAsync(all.data(), xch.p + 128, 128ull * e->nranks, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	long long ok = mine.ok;
	for (int r = 0; r < e->nranks && ok; r++) {
		const PeerInfo &pi = all[r];
		if (!pi.ok || pi.host_hash != mine.host_hash) { ok = 0; break; }           // peer memory needs one NVLink domain: same box
		if (r == e->rank) { e->peer_base[r] = e->peer_block; continue; }
		if (pi.pid == mine.pid) {
			// another handle of this process (one Electron main process driving several GPUs): plain peer access
			int can = 0;
			if (cudaDeviceCanAccessPeer(&can, e->device, pi.device) != cudaSuccess || !can) { cudaGetLastError(); ok = 0; break; }
			const cudaError_t pe = cudaDeviceEnablePeerAccess(pi.device, 0);
			if (pe != cudaSuccess && pe != cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); ok = 0; break; }
			cudaGetLastError();
			e->peer_base[r] = (void *)(uintptr_t)pi.ptr;
		} else {
			void *p = nullptr;
			if (cudaIpcOpenMemHandle(&p, pi.handle, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); ok = 0; break; }
			e->peer_base[r] = p; e->peer_ipc[r] = true;
		}
	}
	// touch every peer's block once now: lazily enabled peer mappings are established on first access, which must not be the first join
	if (ok) {
		for (int r = 0; r < e->nranks; r++)
			if (r != e->rank && apo::run_touch(e->peer_base[r], bytes, xch.p, e->stream) != cudaSuccess) { cudaGetLastError(); ok = 0; break; }
		if (cudaStreamSynchronize(e->stream) != cudaSuccess) { cudaGetLastError(); ok = 0; }
	}
	// agree on the outcome (also the barrier that orders every rank's zero-fill before the first join)
	long long *flag = (long long *)xch.p;
	CK(cudaMemcpyAsync(flag, &ok, 8, cudaMemcpyHostToDevice, e->stream));
	rc = g_nccl.AllReduce(flag, flag, 1, kNcclInt64, kNcclMin, e->comm, e->stream);
	if (rc != 0) { return fail(e, APO_E_NCCL, "ncclAllReduce (peer agreement): %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "error"); }
	CK(cudaMemcpyAsync(&ok, flag, 8, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	if (!ok) { peer_teardown(e); return APO_OK; }
	e->peer_ok = true; e->peer_slot_words = slot_words; e->join_epoch = 0;
	return APO_OK;
}
}  // namespace

// =============================================================================== lifecycle
extern "C" int apo_abi_version(void) { return APO_ABI_VERSION; }

extern "C" int apo_create(int device, apo_engine **out) {
	if (!out) return fail(nullptr, APO_E_ARG, "out is NULL");
	*out = nullptr;
	int n = 0;
	cudaError_t c = cudaGetDeviceCount(&n);
	if (c != cudaSuccess || n == 0)
		return fail(nullptr, APO_E_CUDA, "no CUDA device: %s (this library has no CPU fallback)", c != cudaSuccess ? cudaGetErrorString(c) : "device count is 0");
	if (device < 0 || device >= n) return fail(nullptr, APO_E_ARG, "device %d out of range [0,%d)", device, n);
	apo_engine *e = new (std::nothrow) apo_engine();
	if (!e) return fail(nullptr, APO_E_NOMEM, "out of host memory");
	e->device = device;
	auto bail = [&](const char *what, cudaError_t ce) { fail(nullptr, APO_E_CUDA, "%s: %s", what, cudaGetErrorString(ce)); apo_destroy(e); return APO_E_CUDA; };
	if ((c = cudaSetDevice(device)) != cudaSuccess) return bail("cudaSetDevice", c);
	cudaDeviceProp prop;
	if ((c = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) return bail("cudaGetDeviceProperties", c);
	if (prop.major != 9 || prop.minor != 0) { fail(nullptr, APO_E_CUDA, "device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major, prop.minor); apo_destroy(e); return APO_E_CUDA; }
	e->sm_count = prop.multiProcessorCount;
	e->mem_pitch_max = prop.memPitch;
	{
		// fuse heuristic (apo_score): the corpus scan rides on one warp per SM and must hide behind the evaluation stream.
		// Stream rate = 0.9 x the pin bandwidth of this device for Form D / R (0.61 x for the SM-bound compact layout, kWordFracOfPin
		// x for Form W words); scan rate = kScanRecordsPerSmCycle records per SM clock on that one warp.  Both only steer the fuse /
		// no-fuse choice.
		int mem_khz = 0, bus_bits = 0, sm_khz = 0;
		cudaDeviceGetAttribute(&mem_khz, cudaDevAttrMemoryClockRate, device);
		cudaDeviceGetAttribute(&bus_bits, cudaDevAttrGlobalMemoryBusWidth, device);
		cudaDeviceGetAttribute(&sm_khz, cudaDevAttrClockRate, device);
		constexpr double kStreamFracOfPin = 0.90, kCompactFracOfPin = 0.61, kWordFracOfPin = 0.65 /* K1q on Form W: 2.19 TB/s of 3.35 on an H100 80GB HBM3 at 400 W */, kScanRecordsPerSmCycle = 1.0264e-2;
		if (mem_khz > 0 && bus_bits > 0) {
			const double pin_bytes_per_ms = 2.0 * (double)mem_khz * (double)bus_bits / 8.0;     // kHz x bytes = bytes per ms
			e->stream_bytes_per_ms = kStreamFracOfPin * pin_bytes_per_ms;
			e->stream_q_bytes_per_ms = kCompactFracOfPin * pin_bytes_per_ms;
			e->stream_w_bytes_per_ms = kWordFracOfPin * pin_bytes_per_ms;
		}
		if (sm_khz > 0) e->scan_ms_per_record = 1.0 / (kScanRecordsPerSmCycle * (double)e->sm_count * (double)sm_khz);
	}
	// experiment / test switches: the environment gives the initial value once per handle (never read per call), apo_set_tuning changes them
	e->env_no_fuse = getenv("APO_NO_FUSE") != nullptr;
	e->env_force_fuse = getenv("APO_FORCE_FUSE") != nullptr;
	e->env_no_staging = getenv("APO_NO_STAGING") != nullptr;
	e->env_nccl_join = getenv("APO_JOIN_NCCL") != nullptr;
	e->env_no_twin = getenv("APO_NO_TWIN") != nullptr;
	e->env_no_twin_t = getenv("APO_NO_TWIN_T") != nullptr;
	e->env_twin_t = getenv("APO_TWIN_T") != nullptr;
	e->env_no_twin_t2 = getenv("APO_NO_TWIN_T2") != nullptr;
	if ((c =cudaStreamCreateWithFlags(&e->own_stream, cudaStreamNonBlocking)) != cudaSuccess) return bail("cudaStreamCreate", c);
	if ((c = cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking)) != cudaSuccess) return bail("cudaStreamCreate", c);
	e->stream = e->own_stream;
	for (auto &ev : e->ev) if ((c = cudaEventCreate(&ev)) != cudaSuccess) return bail("cudaEventCreate", c);
	for (int i = 0; i < 2; i++) {
		if ((c = cudaEventCreateWithFlags(&e->win_free[i], cudaEventDisableTiming)) != cudaSuccess) return bail("cudaEventCreate", c);
		if ((c = cudaEventCreateWithFlags(&e->win_ready[i], cudaEventDisableTiming)) != cudaSuccess) return bail("cudaEventCreate", c);
		if ((c = cudaEventCreateWithFlags(&e->stage_done[i], cudaEventDisableTiming)) != cudaSuccess) return bail("cudaEventCreate", c);
	}
	if ((c = cudaMallocHost((void **)&e->h_domain, sizeof(uint32_t))) != cudaSuccess) return bail("cudaMallocHost", c);
	*e->h_domain = 0u;
	memcpy(e->W.w, kDefaultWeights, sizeof kDefaultWeights);
	build_luts(e);
	if (upload_luts(e) != APO_OK) { g_create_error = e->err; apo_destroy(e); return APO_E_CUDA; }
	*out = e;
	return APO_OK;
}

extern "C" void apo_destroy(apo_engine *e) {
	if (!e) return;
	cudaSetDevice(e->device);
	if (e->own_stream) cudaStreamSynchronize(e->own_stream);
	peer_teardown(e);
	if (e->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(e->comm);
	if (e->zc_host) cudaFreeHost(e->zc_host);
	e->q8.release(); e->qd2.release(); e->qli.release(); e->qw.release(); e->qbook.release(); e->d_d2book.release(); e->d_d2stream.release(); e->unpack_bad.release(); e->stage.release();
	e->qt.release(); e->qt_stream.release();
	e->d_lut.release(); e->corpus.release(); e->dims.release(); e->roll.release(); e->acc.release(); e->acc_joined.release(); e->acc_snapshot.release(); e->misc.release();
	e->result.release(); e->keys.release(); e->sel_key.release(); e->sel_idx.release();
	e->cand_acc.release(); e->cand_rep.release(); e->cand_book.release(); e->ccorp_acc.release(); e->ccorp_rep.release();
	e->tup.release(); e->tups.release(); e->tvals.release(); e->tcopy.release();
	e->win[0].release(); e->win[1].release(); e->batch_in.release(); e->batch_out.release(); e->batch_mask.release();
	if (e->h_result) cudaFreeHost(e->h_result);
	if (e->h_domain) cudaFreeHost((void *)e->h_domain);
	for (auto &ev : e->ev) if (ev) cudaEventDestroy(ev);
	for (auto &ev : e->k1_ev) cudaEventDestroy(ev);
	for (int i = 0; i < 2; i++) { if (e->win_free[i]) cudaEventDestroy(e->win_free[i]); if (e->win_ready[i]) cudaEventDestroy(e->win_ready[i]); }
	for (int i = 0; i < 2; i++) { if (e->stage_done[i]) cudaEventDestroy(e->stage_done[i]); if (e->h_stage[i]) cudaFreeHost(e->h_stage[i]); }
	if (e->own_stream) cudaStreamDestroy(e->own_stream);
	if (e->copy_stream) cudaStreamDestroy(e->copy_stream);
	delete e;
}

extern "C" const char *apo_last_error(const apo_engine *e) { return e ? e->err.c_str() : g_create_error.c_str(); }

extern "C" int apo_set_stream(apo_engine *e, uint64_t cuda_stream) {
	if (!e) return APO_E_ARG;
	e->stream = cuda_stream ? (cudaStream_t)(uintptr_t)cuda_stream : e->own_stream;
	return APO_OK;
}

extern "C" int apo_set_tuning(apo_engine *e, uint32_t flags) {
	if (!e) return APO_E_ARG;
	if (flags & ~(APO_TUNE_NO_FUSE | APO_TUNE_FORCE_FUSE | APO_TUNE_NO_STAGING | APO_TUNE_NCCL_JOIN | APO_TUNE_NO_TWIN | APO_TUNE_NO_TWIN_T | APO_TUNE_TWIN_T |
	              APO_TUNE_NO_TWIN_T2))
		return fail(e, APO_E_ARG, "unknown tuning flag %#x", flags);
	e->env_no_fuse = (flags & APO_TUNE_NO_FUSE) != 0; e->env_force_fuse = (flags & APO_TUNE_FORCE_FUSE) != 0;
	e->env_no_staging = (flags & APO_TUNE_NO_STAGING) != 0; e->env_nccl_join = (flags & APO_TUNE_NCCL_JOIN) != 0;
	e->env_no_twin = (flags & APO_TUNE_NO_TWIN) != 0;
	e->env_no_twin_t = (flags & APO_TUNE_NO_TWIN_T) != 0; e->env_twin_t = (flags & APO_TUNE_TWIN_T) != 0;
	e->env_no_twin_t2 = (flags & APO_TUNE_NO_TWIN_T2) != 0;
	return APO_OK;
}

extern "C" int apo_set_weights(apo_engine *e, const double w[APO_NDIM]) {
	if (!e || !w) return fail(e, APO_E_ARG, "NULL argument");
	for (int i = 0; i < APO_NDIM; i++)
		if (!std::isfinite(w[i]) || !(w[i] == 0.0 || (w[i] >= 1e-100 && w[i] <= 1e100)))
			return fail(e, APO_E_ARG, "weights must be 0 or within [1e-100, 1e100]");
	CK(cudaSetDevice(e->device));
	memcpy(e->W.w, w, sizeof e->W.w);
	e->weights_gen++;
	build_luts(e);
	int rc = upload_luts(e);
	if (rc == APO_OK && (e->compact || e->twin)) rc = load_qtables(e, e->qt, e->qt.book);
	e->tcopy.vals.ok[0] = e->tcopy.vals.ok[1] = 0;          // the Form T copy's values belonged to the old weights
	if (rc == APO_OK && e->tcopy.C) rc = tuple_values(e, e->tcopy, e->tcopy.vals, false);
	return rc;
}

extern "C" int apo_get_weights(const apo_engine *e, double w[APO_NDIM]) {
	if (!e || !w) return APO_E_ARG;
	memcpy(w, e->W.w, sizeof e->W.w);
	return APO_OK;
}

// =============================================================================== single-trace path
extern "C" int apo_reward_batch(apo_engine *e, const apo_record *recs, uint64_t n, double *dims, uint32_t *masks, double *finals) {
	if (!e) return APO_E_ARG;
	if (n == 0) return APO_OK;
	if (!recs) return fail(e, APO_E_ARG, "recs is NULL");
	CK(cudaSetDevice(e->device));
	constexpr uint64_t kZeroCopyMax = 1024;      // records: the IDE scores one trace at a time (TCS:408-418, 547)
	if (n <= kZeroCopyMax) {
		// single-trace path: one launch, no copies — the kernel reads the records from and writes the results to one
		// page-locked, device-mapped block (PCIe round trips of a few hundred bytes beat four cudaMemcpyAsync calls)
		const uint64_t per = sizeof(apo_record) + APO_NDIM * 8 + 8 + 4;
		if (!e->zc_host) { CK(cudaMallocHost((void **)&e->zc_host, kZeroCopyMax * per)); e->zc_cap = kZeroCopyMax * per; }
		apo_record *zin = (apo_record *)e->zc_host;
		double *zdims = (double *)(e->zc_host + kZeroCopyMax * sizeof(apo_record));
		double *zfin = zdims + kZeroCopyMax * APO_NDIM;
		uint32_t *zmask = (uint32_t *)(zfin + kZeroCopyMax);
		memcpy(zin, recs, n * sizeof(apo_record));
		CK(apo::run_reward_batch(zin, n, e->W, e->d_lut.p, zdims, zmask, zfin, e->stream));
		CK(cudaStreamSynchronize(e->stream));
		if (dims) memcpy(dims, zdims, n * APO_NDIM * 8);
		if (masks) memcpy(masks, zmask, n * 4);
		if (finals) memcpy(finals, zfin, n * 8);
		return APO_OK;
	}
	CK(reserve(e, e->batch_in, n));
	CK(reserve(e, e->batch_out, n * (APO_NDIM + 1)));
	CK(reserve(e, e->batch_mask, n));
	CK(cudaMemcpyAsync(e->batch_in.p, recs, n * sizeof(apo_record), cudaMemcpyHostToDevice, e->stream));
	CK(apo::run_reward_batch(e->batch_in.p, n, e->W, e->d_lut.p, e->batch_out.p, e->batch_mask.p, e->batch_out.p + n * APO_NDIM, e->stream));
	if (dims) CK(cudaMemcpyAsync(dims, e->batch_out.p, n * APO_NDIM * 8, cudaMemcpyDeviceToHost, e->stream));
	if (masks) CK(cudaMemcpyAsync(masks, e->batch_mask.p, n * 4, cudaMemcpyDeviceToHost, e->stream));
	if (finals) CK(cudaMemcpyAsync(finals, e->batch_out.p + n * APO_NDIM, n * 8, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	return APO_OK;
}

extern "C" int apo_reward_one(apo_engine *e, const apo_record *rec, double dims[APO_NDIM], uint32_t *mask, double *final_reward) {
	return apo_reward_batch(e, rec, 1, dims, mask, final_reward);
}

// =============================================================================== corpus
extern "C" int apo_corpus_upload(apo_engine *e, const apo_record *recs, uint64_t T, uint64_t idx_base) {
	if (!e) return APO_E_ARG;
	if (T && !recs) return fail(e, APO_E_ARG, "recs is NULL");
	CK(cudaSetDevice(e->device));
	CK(reserve(e, e->corpus, T ? T : 1));
	if (T) { const int rc = h2d_rows(e, e->corpus.p, T * sizeof(apo_record), recs, T * sizeof(apo_record), T * sizeof(apo_record), 1, e->stream); if (rc) return rc; }
	CK(apo::run_fill_durclass(e->corpus.p, 32, T, e->stream));        // resident records always carry the duration class
	CK(cudaStreamSynchronize(e->stream));
	e->corpus_T = T; e->corpus_base = idx_base;
	return APO_OK;
}

extern "C" int apo_corpus_upload_json(apo_engine *e, const char *json, uint64_t len, uint64_t idx_base, uint64_t *n_records) {
	if (!e) return APO_E_ARG;
	if (!json) return fail(e, APO_E_ARG, "json is NULL");
	std::vector<apo_record> recs;
	uint64_t pos = 0;
	int64_t n;
	try {
		recs.resize(len / 256 + 16);                      // a persisted trace is never shorter than ~300 bytes
		n = apo_records_from_json(json, len, recs.data(), recs.size(), &pos);
		if (n >= 0 && uint64_t(n) > recs.size()) {
			recs.resize(size_t(n));
			n = apo_records_from_json(json, len, recs.data(), recs.size(), &pos);
		}
	} catch (const std::bad_alloc &) {
		return fail(e, APO_E_NOMEM, "host allocation for %llu bytes of JSON failed", (unsigned long long)len);
	}
	if (n < 0) return fail(e, APO_E_ARG, "malformed trace JSON at byte %llu", (unsigned long long)pos);
	if (n_records) *n_records = uint64_t(n);
	return apo_corpus_upload(e, recs.data(), uint64_t(n), idx_base);
}

extern "C" int apo_corpus_generate(apo_engine *e, uint64_t seed, uint64_t t0, uint64_t T, uint32_t agent_permille) {
	if (!e) return APO_E_ARG;
	CK(cudaSetDevice(e->device));
	CK(reserve(e, e->corpus, T ? T : 1));
	CK(apo::run_gen_records(e->corpus.p, T, seed, 1u, 0, 1, t0, T, agent_permille, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	e->corpus_T = T; e->corpus_base = t0;
	return APO_OK;
}

extern "C" int apo_corpus_download(apo_engine *e, apo_record *out, uint64_t first, uint64_t n) {
	if (!e || !out) return fail(e, APO_E_ARG, "NULL argument");
	if (first + n > e->corpus_T) return fail(e, APO_E_ARG, "range outside the corpus");
	CK(cudaSetDevice(e->device));
	CK(cudaMemcpyAsync(out, e->corpus.p + first, n * sizeof(apo_record), cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	return APO_OK;
}

// =============================================================================== evaluations
extern "C" int apo_dims_upload(apo_engine *e, const float *dims, uint32_t C, uint64_t T) {
	if (!e) return APO_E_ARG;
	if (C && T && !dims) return fail(e, APO_E_ARG, "dims is NULL");
	CK(cudaSetDevice(e->device));
	drop_twin(e);
	const uint64_t pitch = round_up(T ? T : 1, 32);
	CK(reserve(e, e->dims, (uint64_t)(C ? C : 1) * pitch * APO_NDIM));
	if (C && T) {
		// pad evaluations of every row are all-NaN = finalReward null
		if (pitch != T) CK(cudaMemsetAsync(e->dims.p, 0xFF, (uint64_t)C * pitch * APO_NDIM * 4, e->stream));
		{ const int rc = h2d_rows(e, e->dims.p, pitch * APO_NDIM * 4, dims, T * APO_NDIM * 4, T * APO_NDIM * 4, C, e->stream); if (rc) return rc; }
	}
	CK(cudaStreamSynchronize(e->stream));
	e->dims_ptr = e->dims.p; e->dims_C = C; e->dims_T = T; e->dims_pitch = pitch; e->compact = false;
	return build_twin(e);
}

extern "C" int apo_dims_generate(apo_engine *e, uint64_t seed, uint32_t c0, uint32_t C, uint64_t t0, uint64_t T, uint32_t agent_permille) {
	if (!e) return APO_E_ARG;
	CK(cudaSetDevice(e->device));
	drop_twin(e);
	const uint64_t pitch = round_up(T ? T : 1, 32);
	CK(reserve(e, e->dims, (uint64_t)(C ? C : 1) * pitch * APO_NDIM));
	if (pitch != T && C) CK(cudaMemsetAsync(e->dims.p, 0xFF, (uint64_t)C * pitch * APO_NDIM * 4, e->stream));
	CK(apo::run_gen_dims(e->dims.p, pitch, seed, c0, C, t0, T, agent_permille, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	e->dims_ptr = e->dims.p; e->dims_C = C; e->dims_T = T; e->dims_pitch = pitch; e->compact = false;
	return build_twin(e);
}

extern "C" int apo_dims_download(apo_engine *e, float *out, uint32_t c, uint64_t first, uint64_t n) {
	if (!e || !out) return fail(e, APO_E_ARG, "NULL argument");
	if ((!e->dims_ptr && !e->compact) || c >= e->dims_C || first + n > e->dims_T) return fail(e, APO_E_ARG, "range outside the evaluations");
	CK(cudaSetDevice(e->device));
	if (e->compact) {
		CK(reserve(e, e->stage, (n ? n : 1) * APO_NDIM));
		const uint64_t off = (uint64_t)c * e->dims_pitch + first;
		CK(apo::run_decode(e->q8.p + off, e->qd2.p + off, e->qli.p + off, n, e->qbook.p, e->stage.p, e->stream));
		CK(cudaMemcpyAsync(out, e->stage.p, n * APO_NDIM * 4, cudaMemcpyDeviceToHost, e->stream));
		CK(cudaStreamSynchronize(e->stream));
		return APO_OK;
	}
	CK(cudaMemcpyAsync(out, e->dims_ptr + ((uint64_t)c * e->dims_pitch + first) * APO_NDIM, n * APO_NDIM * 4, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	return APO_OK;
}

extern "C" int apo_dims_attach(apo_engine *e, uint64_t device_ptr, uint32_t C, uint64_t T, uint64_t pitch_evals) {
	if (!e) return APO_E_ARG;
	if (!device_ptr || device_ptr % 16) return fail(e, APO_E_ARG, "device pointer must be non-NULL and 16-byte aligned");
	if (pitch_evals % 4 || pitch_evals < round_up(T, 4)) return fail(e, APO_E_ARG, "pitch must be a multiple of 4 evaluations and >= T rounded up to 4");
	drop_twin(e);                                       // never a copy of caller-owned memory: the caller may change it
	e->dims_ptr = (const float *)(uintptr_t)device_ptr; e->dims_C = C; e->dims_T = T; e->dims_pitch = pitch_evals; e->compact = false;
	return APO_OK;
}

extern "C" int apo_dims_layout(const apo_engine *e) {
	if (!e) return 0;
	if (e->compact) return 2;
	return (e->dims_ptr && e->dims_C) ? 1 : 0;
}

extern "C" int apo_dims_compact(apo_engine *e) {
	if (!e) return APO_E_ARG;
	if (e->compact) return APO_OK;
	if (!e->dims_ptr || e->dims_C == 0) return fail(e, APO_E_STATE, "no dims loaded");
	CK(cudaSetDevice(e->device));
	if (e->twin && !e->twin_w) {                        // the copy built at load already is this tensor in Form Q
		e->tcopy.release();                             // a compact tensor keeps no Form T copy
		e->twin = false; e->compact = true; e->dims_ptr = nullptr;
		e->dims.release();
		return APO_OK;
	}
	drop_twin(e);                                       // a Form W copy is not a compact tensor: transcode the fp32 one
	const uint32_t C = e->dims_C; const uint64_t T = e->dims_T, pitch_in = e->dims_pitch, pitch = round_up(T ? T : 1, 32);
	int rc = compact_begin(e, C, pitch);
	if (rc) return rc;
	CK(apo::run_transcode(e->dims_ptr, pitch_in, C, T, e->q8.p, e->qd2.p, pitch, e->qbook.p, e->qbook.p + 8 * 256, e->stream));
	const float *keep = e->dims_ptr;
	if ((rc = compact_finish(e, C, T, pitch))) { e->dims_ptr = keep; return rc; }
	e->dims.release();                                  // the fp32 copy (if engine-owned) is no longer needed
	return APO_OK;
}

namespace {
// chunked producer -> transcoder: at most ~2 GB of fp32 staging, never the whole tensor
template <class Fill>
int compact_stream(apo_engine *e, uint32_t C, uint64_t T, Fill fill) {
	CK(cudaSetDevice(e->device));
	drop_twin(e);
	const uint64_t pitch = round_up(T ? T : 1, 32);
	uint64_t Cc = (2ull << 30) / (pitch * 36);
	if (Cc < 1) Cc = 1;
	if (Cc > C) Cc = C ? C : 1;
	CK(reserve(e, e->stage, Cc * pitch * APO_NDIM));
	int rc = compact_begin(e, C, pitch);
	if (rc) return rc;
	for (uint32_t c0 = 0; c0 < C; c0 += (uint32_t)Cc) {
		const uint32_t cn = C - c0 < Cc ? C - c0 : (uint32_t)Cc;
		if ((rc = fill(c0, cn, e->stage.p, pitch))) return rc;
		CK(apo::run_transcode(e->stage.p, pitch, cn, T, e->q8.p + (uint64_t)c0 * pitch, e->qd2.p + (uint64_t)c0 * pitch, pitch,
		                      e->qbook.p, e->qbook.p + 8 * 256, e->stream));
	}
	e->compact = false; e->dims_ptr = nullptr; e->dims_C = 0;          // whatever was loaded before is superseded
	rc = compact_finish(e, C, T, pitch);
	e->stage.release();
	if (rc == APO_OK) e->dims.release();
	return rc;
}
}  // namespace

extern "C" int apo_dims_generate_compact(apo_engine *e, uint64_t seed, uint32_t c0, uint32_t C, uint64_t t0, uint64_t T, uint32_t agent_permille) {
	if (!e) return APO_E_ARG;
	return compact_stream(e, C, T, [&](uint32_t cb, uint32_t cn, float *stage, uint64_t pitch) -> int {
		CK(apo::run_gen_dims(stage, pitch, seed, c0 + cb, cn, t0, T, agent_permille, e->stream));
		return APO_OK;
	});
}

extern "C" int apo_dims_upload_compact(apo_engine *e, const float *dims, uint32_t C, uint64_t T) {
	if (!e) return APO_E_ARG;
	if (C && T && !dims) return fail(e, APO_E_ARG, "dims is NULL");
	return compact_stream(e, C, T, [&](uint32_t cb, uint32_t cn, float *stage, uint64_t pitch) -> int {
		const int rc = h2d_rows(e, stage, pitch * APO_NDIM * 4, dims + (uint64_t)cb * T * APO_NDIM, T * APO_NDIM * 4, T * APO_NDIM * 4, cn, e->stream);
		if (rc) return rc;
		CK(cudaStreamSynchronize(e->stream));              // the host chunk may be reused by the caller after return
		return APO_OK;
	});
}

namespace {
int rollouts_upload_rows(apo_engine *e, const void *recs, uint32_t row, uint32_t C, uint64_t T) {
	if (!e) return APO_E_ARG;
	if (C && T && !recs) return fail(e, APO_E_ARG, "recs is NULL");
	CK(cudaSetDevice(e->device));
	const uint64_t pitch = round_up(T ? T : 1, 4);
	CK(reserve(e, e->roll, (uint64_t)(C ? C : 1) * pitch * row));
	if (C && T) {
		if (pitch != T) CK(cudaMemsetAsync(e->roll.p, 0, (uint64_t)C * pitch * row, e->stream));   // VALID clear
		{ const int rc = h2d_rows(e, e->roll.p, pitch * row, recs, T * row, T * row, C, e->stream); if (rc) return rc; }
		CK(apo::run_fill_durclass(e->roll.p, row, (uint64_t)C * pitch, e->stream));
	}
	CK(cudaStreamSynchronize(e->stream));
	e->roll_C = C; e->roll_T = T; e->roll_pitch = pitch; e->roll_row = row;
	return APO_OK;
}
int rollouts_generate_rows(apo_engine *e, uint32_t row, uint64_t seed, uint32_t c0, uint32_t C, uint64_t t0, uint64_t T, uint32_t agent_permille) {
	if (!e) return APO_E_ARG;
	CK(cudaSetDevice(e->device));
	const uint64_t pitch = round_up(T ? T : 1, 4);
	CK(reserve(e, e->roll, (uint64_t)(C ? C : 1) * pitch * row));
	if (pitch != T && C) CK(cudaMemsetAsync(e->roll.p, 0, (uint64_t)C * pitch * row, e->stream));
	if (row == 32) CK(apo::run_gen_records((apo_record *)e->roll.p, pitch, seed, 2u, c0, C, t0, T, agent_permille, e->stream));
	else CK(apo::run_gen_records16((apo_record16 *)e->roll.p, pitch, seed, 2u, c0, C, t0, T, agent_permille, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	e->roll_C = C; e->roll_T = T; e->roll_pitch = pitch; e->roll_row = row;
	return APO_OK;
}
int rollouts_download_rows(apo_engine *e, void *out, uint32_t row, uint32_t c, uint64_t first, uint64_t n) {
	if (!e || !out) return fail(e, APO_E_ARG, "NULL argument");
	if (!e->roll.p || e->roll_row != row) return fail(e, APO_E_STATE, "no rollouts of that row size loaded");
	if (c >= e->roll_C || first + n > e->roll_T) return fail(e, APO_E_ARG, "range outside the rollouts");
	CK(cudaSetDevice(e->device));
	CK(cudaMemcpyAsync(out, e->roll.p + ((uint64_t)c * e->roll_pitch + first) * row, n * row, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	return APO_OK;
}
}  // namespace

extern "C" int apo_rollouts_upload(apo_engine *e, const apo_record *recs, uint32_t C, uint64_t T) { return rollouts_upload_rows(e, recs, 32, C, T); }
extern "C" int apo_rollouts16_upload(apo_engine *e, const apo_record16 *recs, uint32_t C, uint64_t T) { return rollouts_upload_rows(e, recs, 16, C, T); }
extern "C" int apo_rollouts_generate(apo_engine *e, uint64_t seed, uint32_t c0, uint32_t C, uint64_t t0, uint64_t T, uint32_t agent_permille) {
	return rollouts_generate_rows(e, 32, seed, c0, C, t0, T, agent_permille);
}
extern "C" int apo_rollouts16_generate(apo_engine *e, uint64_t seed, uint32_t c0, uint32_t C, uint64_t t0, uint64_t T, uint32_t agent_permille) {
	return rollouts_generate_rows(e, 16, seed, c0, C, t0, T, agent_permille);
}
extern "C" int apo_rollouts_download(apo_engine *e, apo_record *out, uint32_t c, uint64_t first, uint64_t n) { return rollouts_download_rows(e, out, 32, c, first, n); }
extern "C" int apo_rollouts16_download(apo_engine *e, apo_record16 *out, uint32_t c, uint64_t first, uint64_t n) { return rollouts_download_rows(e, out, 16, c, first, n); }

extern "C" int apo_record_pack16(const apo_record *in, uint64_t n, apo_record16 *out, uint64_t *bad) {
	if ((!in || !out) && n) return APO_E_ARG;
	for (uint64_t i = 0; i < n; i++) {
		if (!apo::representable16(in[i])) { if (bad) *bad = i; return APO_E_ARG; }
		out[i] = apo::pack16(in[i]);
	}
	return APO_OK;
}
extern "C" int apo_record_unpack16(const apo_record16 *in, uint64_t n, apo_record *out) {
	if ((!in || !out) && n) return APO_E_ARG;
	for (uint64_t i = 0; i < n; i++) out[i] = apo::unpack16(in[i]);
	return APO_OK;
}

// =============================================================================== scoring
extern "C" int apo_score_begin(apo_engine *e, uint32_t C_total) {
	if (!e) return APO_E_ARG;
	if (C_total == 0) return fail(e, APO_E_ARG, "C_total is 0");
	CK(cudaSetDevice(e->device));
	int rc = ensure_scratch(e, C_total, C_total);
	if (rc) return rc;
	e->timing_on = true;
	return begin_score(e, C_total);
}

extern "C" int apo_score_accumulate(apo_engine *e, const apo_score_opts *o, uint32_t cand_offset) {
	if (!e) return APO_E_ARG;
	if (!e->scoring) return fail(e, APO_E_STATE, "apo_score_begin has not been called");
	Evals ev;
	int rc = resident_evals(e, o, &ev);
	if (rc) return rc;
	if ((uint64_t)cand_offset + ev.C > e->score_C) return fail(e, APO_E_ARG, "candidates [%u,%u) exceed C_total=%u", cand_offset, cand_offset + ev.C, e->score_C);
	if ((rc = check_window(e, o, ev.count))) return rc;
	const bool cand = wants_cand(o), ccorp = wants_ccorp(o);
	if (cand && (rc = cand_check(e))) return rc;
	if (ccorp && (rc = ccorp_check(e, ev.records()))) return rc;
	CK(cudaSetDevice(e->device));
	if (cand && (rc = cand_reserve(e, e->score_C))) return rc;                                  // allocates: before route_twin
	if (cand && e->cand_every && !e->cand_armed && (rc = cand_arm(e, e->score_C))) return rc;
	if ((rc = twin_t_ready(e, o))) return rc;
	route_twin(e, o, &ev);
	if ((rc = resident_window(e, o, &ev)) || (rc = launch_score(e, o, ev, cand_offset))) return rc;
	if (!ccorp) e->ccorp_every = false;
	else if (e->ccorp_every) {                          // an earlier accumulate of the session did not set the flag: finish refuses
		if (!e->ccorp_armed && (rc = ccorp_arm(e, e->score_C))) return rc;
		if ((rc = launch_ccorp(e, ev, cand_offset))) return rc;
	}
	if (!cand) { e->cand_every = false; return APO_OK; }
	if (!e->cand_every) return APO_OK;                  // an earlier accumulate of the session did not set the flag: finish refuses
	return launch_cand(e, ev, cand_offset);
}

extern "C" int apo_score_finish(apo_engine *e, const apo_score_opts *o, double *scores, uint64_t *counts, int32_t *topk,
                                apo_corpus_report *report) {
	if (!e) return APO_E_ARG;
	e->cand_ready = e->ccorp_ready = false;             // a failed finish leaves no breakdown behind either
	if (!o) return fail(e, APO_E_ARG, "opts is NULL");
	if (!e->scoring) return fail(e, APO_E_STATE, "apo_score_begin has not been called");
	int rc = score_check(e, o, e->score_C, kSession, true);      // the accumulate calls refused every other source
	if (rc) return rc;
	if (wants_cand(o) && !e->cand_every)
		return fail(e, APO_E_STATE, "APO_SCORE_CANDIDATES: every apo_score_accumulate of the session must set the flag for a breakdown");
	if (wants_ccorp(o) && !e->ccorp_every)
		return fail(e, APO_E_STATE, "APO_SCORE_CANDIDATE_CORPUS: every apo_score_accumulate of the session must set the flag for the reports");
	if ((rc = score_arm(e, o, e->score_C, false))) return rc;   // nothing accumulated yet: an empty breakdown
	return finish_score(e, o, e->score_C, scores, counts, topk, report);
}

extern "C" int apo_score(apo_engine *e, const apo_score_opts *o, double *scores, uint64_t *counts, int32_t *topk, apo_corpus_report *report) {
	if (!e) return APO_E_ARG;
	e->cand_ready = e->ccorp_ready = false;             // a failed call leaves no breakdown behind either
	Evals ev;
	int rc = resident_evals(e, o, &ev);
	if (rc) return rc;
	const uint32_t C = ev.C;
	if ((rc = score_check(e, o, C, ev.count, ev.records())) || (rc = twin_t_ready(e, o))) return rc;
	route_twin(e, o, &ev);
	if ((rc = resident_window(e, o, &ev))) return rc;
	const bool tup = ev.form == apo::CAND_T;            // gather-and-add kernel: stand-alone corpus scan + tail
	const double stream_bytes = (double)C * (double)ev.count * ev.bytes();
	// One launch per call: the corpus scan (K2) rides on an extra warp of every scoring CTA and the last CTA finalises (K3,
	// after the peer-memory join when the record axis is sharded) ... when the scan can hide behind the evaluation stream.
	// Both rates are derived from the device at apo_create.
	const double k1_ms = stream_bytes / (ev.form == apo::CAND_Q ? e->stream_q_bytes_per_ms
	                                     : ev.form == apo::CAND_W ? e->stream_w_bytes_per_ms : e->stream_bytes_per_ms);
	const double scan_ms = (double)e->corpus_T * e->scan_ms_per_record;
	const bool one_launch = e->nranks == 1 || peer_join_active(e, C);
	// ... or when it is tiny anyway (the IDE's real corpora, <= 1000 traces): at most 16 records per lane of the corpus warps,
	// a few microseconds, against a second launch
	const uint64_t tiles = (uint64_t)C * ((ev.count + ev.tile() - 1) / ev.tile());
	const uint64_t ctas = tiles < (uint64_t)e->sm_count ? tiles : (uint64_t)e->sm_count;
	const bool small_scan = e->corpus_T <= 16ull * 32ull * ctas;
	const bool fuse = !tup && wants_corpus(e, o) && ev.count > 0 && !e->env_no_fuse && (k1_ms > 1.3 * scan_ms || small_scan || e->env_force_fuse);
	// without a corpus request the same tail still saves the K3 launch: an empty scan, then the last CTA finalises
	const bool tail_only = !tup && !wants_corpus(e, o) && one_launch && ev.count > 0 && !e->env_no_fuse;
	const bool fused = fuse || tail_only;
	if ((rc = score_arm(e, o, C, true, (uint64_t)stream_bytes, fused))) return rc;
	apo::K2Params k2{};
	if (fused) {
		apo::FinalizeParams F = make_fin(e, C, o->K, fuse ? 1 : 0);
		// the finalising CTA is in this launch: it can leave the block zeroed (finish_score records that it did)
		if (one_launch) { F.clean_ptr = e->acc.p; F.clean_words = (uint32_t)(acc_words(C, e->nranks) + ARM_WORDS); F.snapshot = e->acc_snapshot.p; }
		k2 = make_k2(e, C, F);
		if (tail_only) { k2.T = 0; k2.recs = nullptr; }
	}
	if ((rc = launch_score(e, o, ev, 0, fused ? &k2 : nullptr))) return rc;
	if (wants_cand(o) && (rc = launch_cand(e, ev, 0))) return rc;
	if (wants_ccorp(o) && (rc = launch_ccorp(e, ev, 0))) return rc;
	return finish_score(e, o, C, scores, counts, topk, report, fused);
}

namespace {
int tuples_args(apo_engine *e, const uint16_t *tl, const uint8_t *th, const uint32_t *tb_pc, const uint16_t *tb_pd, uint32_t n,
                const uint32_t *codebook, const uint32_t *d2book, uint32_t C, uint64_t T) {
	if (C == 0) return fail(e, APO_E_ARG, "C == 0");
	if (!codebook || !d2book || (n && (!tb_pc || !tb_pd)) || (T && (!tl || !th))) return fail(e, APO_E_ARG, "input is NULL");
	if (n > APO_TUPLES_MAX) return fail(e, APO_E_ARG, "n_tuples=%u exceeds %u", n, APO_TUPLES_MAX);
	if (T && n == 0) return fail(e, APO_E_ARG, "evaluations without a dictionary");
	return APO_OK;
}

// the caller's dictionary of n entries into d (pageable sources are consumed when this returns)
int dict_upload(apo_engine *e, TupleDict &d, const uint32_t *pc, const uint16_t *pd, uint32_t n, const uint32_t *codebook, const uint32_t *d2book) {
	CK(reserve(e, d.pc, n ? n : 1));
	CK(reserve(e, d.pd, n ? n : 1));
	CK(reserve(e, d.d2, 4096));
	if (n) {
		CK(cudaMemcpyAsync(d.pc.p, pc, (uint64_t)n * 4, cudaMemcpyHostToDevice, e->stream));
		CK(cudaMemcpyAsync(d.pd.p, pd, (uint64_t)n * 2, cudaMemcpyHostToDevice, e->stream));
	}
	CK(cudaMemcpyAsync(d.d2.p, d2book, 4096 * 4, cudaMemcpyHostToDevice, e->stream));   // bit patterns: unused slots are NaNs, flagged if an entry names one
	memcpy(d.book, codebook, sizeof d.book);
	d.n = n;
	return APO_OK;
}

// A tensor [C][T] in the caller's memory for the host-streaming calls: the planes of one layout, each [C][T] at `bytes` per
// evaluation.  D / R / R16: the rows; Q: q8, d2, li; P: pc, pd; T: tl, th.
struct HostTensor {
	Form form;                                   // what the scoring kernel reads (Form P: Form Q, which k_unpack_p expands it into)
	uint32_t C;
	uint64_t T;
	struct { const void *p; uint32_t bytes; } plane[3];
	int planes;
	bool packed = false;                         // Form P
	const uint32_t *codebook = nullptr;          // Form Q / P / T
	const uint32_t *d2book = nullptr;            // Form P / T
	const uint32_t *tb_pc = nullptr;             // Form T: the dictionary
	const uint16_t *tb_pd = nullptr;
	uint32_t n_tuples = 0;
};

// Streams a host tensor through two device windows of ~256 MB: the H2D copy of chunk i+1 (copy stream) overlaps the scoring
// kernel and the per-candidate passes on chunk i (compute stream).  A window holds the planes one after the other, [C][Tc] each.
int stream_host(apo_engine *e, const apo_score_opts *o, const HostTensor &h, double *scores, uint64_t *counts, int32_t *topk,
                apo_corpus_report *report) {
	const uint32_t C = h.C;
	const uint64_t T = h.T;
	e->cand_ready = e->ccorp_ready = false;
	if (!o) return fail(e, APO_E_ARG, "opts is NULL");
	const bool rows = h.form != apo::CAND_Q && h.form != apo::CAND_T;
	if (!rows && wants_ccorp(o)) return ccorp_check(e, false);   // the wire formats refuse it before they look at their inputs
	int rc;
	if (h.form == apo::CAND_T) {
		if ((rc = tuples_args(e, (const uint16_t *)h.plane[0].p, (const uint8_t *)h.plane[1].p, h.tb_pc, h.tb_pd, h.n_tuples, h.codebook,
		                      h.d2book, C, T)))
			return rc;
	} else {
		bool missing = C == 0 || (h.form == apo::CAND_Q && !h.codebook) || (h.packed && !h.d2book);
		for (int k = 0; k < h.planes; k++) missing |= h.plane[k].p == nullptr;
		if (missing) return fail(e, APO_E_ARG, "input is NULL or C == 0");
	}
	Evals ev;
	ev.form = h.form; ev.C = C; ev.variant = (int)o->variant;
	if ((rc = score_check(e, o, C, kStreamed, ev.records()))) return rc;
	if (h.form == apo::CAND_Q) {                                   // Form Q / P: K1q's tables of this call's codebook
		if ((rc = load_qtables(e, e->qt_stream, h.codebook))) return rc;
		ev.qt = &e->qt_stream;
		ev.variant = e->qt_stream.pair_ok ? 0 : 4;
	}
	uint64_t wire = 0;                                             // bytes per evaluation over PCIe
	for (int k = 0; k < h.planes; k++) wire += h.plane[k].bytes;
	const uint64_t dev = h.packed ? 14 + wire : wire;             // per window evaluation: Form P also holds the Form Q planes
	// window of ~256 MB per buffer, a multiple of the scoring kernel's tile so chunks never split a tile
	const uint64_t tile = ev.tile();
	uint64_t Tc = (256ull << 20) / ((uint64_t)C * wire);
	Tc = Tc / tile * tile;
	if (Tc < tile) Tc = tile;
	if (Tc > round_up(T ? T : 1, tile)) Tc = round_up(T ? T : 1, tile);
	for (int i = 0; i < 2; i++) CK(reserve(e, e->win[i], (uint64_t)C * Tc * dev));
	// pageable callers (malloc / ArrayBuffer / numpy) of the row formats: the driver would stage such copies through one small
	// internal buffer on the calling thread; instead gather each chunk into pinned memory with a few host threads while the
	// previous chunk is on the wire.  Pinned or registered callers (apo_host_alloc) are read in place.
	const bool staged = rows && T > 0 && is_pageable(h.plane[0].p) && !e->env_no_staging;
	if (staged && (rc = ensure_stage(e, (uint64_t)C * Tc * wire))) return rc;
	uint64_t code_ok[2] = {0, 0};      // Form P: bit 16 j + c set when code c of coded dimension j names a value (not empty, not NaN)
	if (h.packed) {
		for (int j = 0; j < 8; j++)
			for (int c = 0; c < 15; c++) {
				const uint32_t bits = h.codebook[256 * j + c];
				if ((bits & 0x7FFFFFFFu) <= 0x7F800000u) code_ok[j >> 2] |= 1ull << (16 * (j & 3) + c);
			}
		CK(reserve(e, e->d_d2stream, 4096));
		CK(reserve(e, e->unpack_bad, 1));
		CK(cudaMemcpyAsync(e->d_d2stream.p, h.d2book, 4096 * 4, cudaMemcpyHostToDevice, e->stream));   // bit patterns: empty slots are NaNs, flagged if named
		CK(cudaMemsetAsync(e->unpack_bad.p, 0, 4, e->stream));
	}
	if ((rc = score_arm(e, o, C, true, (uint64_t)C * T * wire))) return rc;
	if (h.form == apo::CAND_T) {                                   // the dictionary and its values, once for the whole call
		if (wants_cand(o) && (rc = cand_upload_tbook(e, h.codebook))) return rc;
		if ((rc = dict_upload(e, e->tups, h.tb_pc, h.tb_pd, h.n_tuples, h.codebook, h.d2book))) return rc;
		ev.dict = &e->tups; ev.tv = &e->tvals; ev.t_once = true;
		if ((rc = tuple_values(e, e->tups, e->tvals, (o->flags & APO_SCORE_RECIP) != 0))) return rc;
	}
	const uint64_t CTc = (uint64_t)C * Tc;
	ev.pitch_evals = Tc;
	int nchunk = 0;
	for (uint64_t t0 = 0; t0 < T; t0 += Tc, nchunk++) {
		const int b = nchunk & 1;
		const uint64_t n = T - t0 < Tc ? T - t0 : Tc;
		uint8_t *w = e->win[b].p;
		if (nchunk >= 2) CK(cudaStreamWaitEvent(e->copy_stream, e->win_free[b], 0));
		uint8_t *dst = w + CTc * (dev - wire);                      // Form P: behind the Form Q planes
		for (int k = 0; k < h.planes; k++) {
			const uint64_t pb = h.plane[k].bytes;
			const uint8_t *src = (const uint8_t *)h.plane[k].p + t0 * pb;
			size_t spitch = T * pb;
			if (staged) {
				if (nchunk >= 2) CK(cudaEventSynchronize(e->stage_done[b]));      // the copy that read this staging buffer has finished
				parallel_rows_copy(e->h_stage[b], Tc * pb, src, spitch, n * pb, C);
				src = e->h_stage[b]; spitch = Tc * pb;
			}
			if ((rc = copy_rows_h2d(e, dst, Tc * pb, src, spitch, n * pb, C, e->copy_stream))) return rc;
			dst += CTc * pb;
		}
		if (staged) CK(cudaEventRecord(e->stage_done[b], e->copy_stream));
		CK(cudaEventRecord(e->win_ready[b], e->copy_stream));
		CK(cudaStreamWaitEvent(e->stream, e->win_ready[b], 0));
		ev.count = n; ev.idx_base = t0;
		if (rows) ev.rows = w;
		if (h.form == apo::CAND_Q) { ev.q8 = (const unsigned long long *)w; ev.d2 = (const float *)(w + CTc * 8); ev.li = (const unsigned short *)(w + CTc * 12); }
		if (h.form == apo::CAND_T) { ev.tl = (const unsigned short *)w; ev.th = w + CTc * 2; }
		if (ev.records()) {                                            // trace records: make sure the window carries the duration class
			CK(apo::run_fill_durclass(w, ev.row(), CTc, e->stream));
			e->timing.launches++;
		}
		if (h.packed) {
			CK(apo::run_unpack_p((const uint32_t *)(w + CTc * 14), (const unsigned short *)(w + CTc * 18), Tc, C, n, e->d_d2stream.p, code_ok[0],
			                     code_ok[1], e->unpack_bad.p, (unsigned long long *)w, (float *)(w + CTc * 8), (unsigned short *)(w + CTc * 12), Tc, e->stream));
			e->timing.launches++;
		}
		if ((rc = launch_score(e, o, ev, 0))) return rc;
		if (wants_cand(o) && (rc = launch_cand(e, ev, 0))) return rc;
		if (wants_ccorp(o) && (rc = launch_ccorp(e, ev, 0))) return rc;   // before the window is released
		CK(cudaEventRecord(e->win_free[b], e->stream));
	}
	return finish_score(e, o, C, scores, counts, topk, report, false, h.packed);
}

int score_host(apo_engine *e, const apo_score_opts *o, const HostTensor &h, double *scores, uint64_t *counts, int32_t *topk,
               apo_corpus_report *report) {
	if (!e) return APO_E_ARG;
	const int rc = stream_host(e, o, h, scores, counts, topk, report);
	if (rc) {
		// a failure in the middle of the chunk loop: nothing may still be reading the caller's memory when we return
		cudaStreamSynchronize(e->copy_stream);
		cudaStreamSynchronize(e->stream);
		if (h.form == apo::CAND_T) e->tvals_check = nullptr;
	}
	return rc;
}
}  // namespace

// =============================================================================== Form Q in host memory (compact wire format)
extern "C" int apo_dims_codebook(apo_engine *e, uint32_t *codebook) {
	if (!e || !codebook) return fail(e, APO_E_ARG, "NULL argument");
	if (!e->compact) return fail(e, APO_E_STATE, "no compact (Form Q) evaluations loaded");
	memcpy(codebook, e->qt.book, sizeof e->qt.book);
	return APO_OK;
}

extern "C" int apo_dims_compact_download(apo_engine *e, uint64_t *q8, float *d2, uint16_t *li, uint32_t c, uint64_t first, uint64_t n) {
	if (!e || !q8 || !d2 || !li) return fail(e, APO_E_ARG, "NULL argument");
	if (!e->compact) return fail(e, APO_E_STATE, "no compact (Form Q) evaluations loaded");
	if (c >= e->dims_C || first + n > e->dims_T) return fail(e, APO_E_ARG, "range outside the evaluations");
	CK(cudaSetDevice(e->device));
	const uint64_t off = (uint64_t)c * e->dims_pitch + first;
	CK(cudaMemcpyAsync(q8, e->q8.p + off, n * 8, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaMemcpyAsync(d2, e->qd2.p + off, n * 4, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaMemcpyAsync(li, e->qli.p + off, n * 2, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	return APO_OK;
}

namespace {
// order of a d2book: by value, -0.0 (sign bit set) before +0.0
bool d2_before(uint32_t x, uint32_t y) {
	float fx, fy; memcpy(&fx, &x, 4); memcpy(&fy, &y, 4);
	if (fx != fy) return fx < fy;
	return x > y;
}

// d2book of the resident Form Q tensor: distinct tool_success_rate values ordered by value (built once per loaded tensor)
int ensure_d2book(apo_engine *e) {
	if (e->d2book_n != ~0u) return APO_OK;
	DevBuf<uint32_t> table;
	CK(table.reserve(16384 + 1));
	CK(cudaMemsetAsync(table.p, 0xFF, 16384 * 4, e->stream));
	CK(cudaMemsetAsync(table.p + 16384, 0, 4, e->stream));
	// pad evaluations carry a cleared presence bit, so the whole pitched planes can be scanned
	CK(apo::run_collect_d2(e->qd2.p, e->qli.p, (uint64_t)e->dims_C * e->dims_pitch, table.p, table.p + 16384, e->stream));
	std::vector<uint32_t> host(16384 + 1);
	CK(cudaMemcpyAsync(host.data(), table.p, host.size() * 4, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	table.release();
	if (host[16384] > 4095) return fail(e, APO_E_STATE, "tool_success_rate takes %u distinct values: more than the 4095 Form P can index", host[16384]);
	std::vector<uint32_t> vals;
	for (int i = 0; i < 16384; i++) if (host[i] != 0xFFFFFFFFu) vals.push_back(host[i]);
	std::sort(vals.begin(), vals.end(), d2_before);
	for (size_t c = 0; c < 4096; c++) e->d2book_host[c] = c < vals.size() ? vals[c] : 0xFFFFFFFFu;
	CK(reserve(e, e->d_d2book, 4096));
	CK(cudaMemcpyAsync(e->d_d2book.p, e->d2book_host, 4096 * 4, cudaMemcpyHostToDevice, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	e->d2book_n = (uint32_t)vals.size();
	return APO_OK;
}
}  // namespace

extern "C" int apo_dims_d2book(apo_engine *e, uint32_t *d2book) {
	if (!e || !d2book) return fail(e, APO_E_ARG, "NULL argument");
	if (!e->compact) return fail(e, APO_E_STATE, "no compact (Form Q) evaluations loaded");
	CK(cudaSetDevice(e->device));
	const int rc = ensure_d2book(e);
	if (rc) return rc;
	memcpy(d2book, e->d2book_host, sizeof e->d2book_host);
	return APO_OK;
}

extern "C" int apo_dims_packed_download(apo_engine *e, uint32_t *pc, uint16_t *pd, uint32_t c, uint64_t first, uint64_t n) {
	if (!e || !pc || !pd) return fail(e, APO_E_ARG, "NULL argument");
	if (!e->compact) return fail(e, APO_E_STATE, "no compact (Form Q) evaluations loaded");
	if (c >= e->dims_C || first + n > e->dims_T) return fail(e, APO_E_ARG, "range outside the evaluations");
	CK(cudaSetDevice(e->device));
	int rc = ensure_d2book(e);
	if (rc) return rc;
	if (n == 0) return APO_OK;
	CK(reserve(e, e->stage, (n * 6 + 3) / 4 + 16));
	uint32_t *dpc = (uint32_t *)e->stage.p;
	unsigned short *dpd = (unsigned short *)(dpc + n);
	uint32_t *bad = (uint32_t *)(e->stage.p + (n * 6 + 3) / 4 + 8);
	CK(cudaMemsetAsync(bad, 0, 4, e->stream));
	const uint64_t off = (uint64_t)c * e->dims_pitch + first;
	CK(apo::run_pack_p(e->q8.p + off, e->qd2.p + off, e->qli.p + off, n, (const uint32_t *)e->d_d2book.p, e->d2book_n, dpc, dpd, bad, e->stream));
	uint32_t hbad = 0;
	CK(cudaMemcpyAsync(pc, dpc, n * 4, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaMemcpyAsync(pd, dpd, n * 2, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaMemcpyAsync(&hbad, bad, 4, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	if (hbad) return fail(e, APO_E_STATE, "a coded dimension takes more than 15 distinct values: not representable in Form P");
	return APO_OK;
}

// Form Q planes (8 + 4 + 2 B per evaluation) for callers that hold the compact wire format: 14 B / evaluation over PCIe instead of 36
extern "C" int apo_score_host_compact(apo_engine *e, const apo_score_opts *o, const uint64_t *q8, const float *d2, const uint16_t *li,
                                      const uint32_t *codebook, uint32_t C, uint64_t T, double *scores, uint64_t *counts,
                                      int32_t *topk, apo_corpus_report *report) {
	HostTensor h{apo::CAND_Q, C, T, {{q8, 8}, {d2, 4}, {li, 2}}, 3};
	h.codebook = codebook;
	return score_host(e, o, h, scores, counts, topk, report);
}

// Form P: 6 B per evaluation cross PCIe and k_unpack_p expands each window to Form Q on the device
extern "C" int apo_score_host_packed(apo_engine *e, const apo_score_opts *o, const uint32_t *pc, const uint16_t *pd, const uint32_t *codebook,
                                     const uint32_t *d2book, uint32_t C, uint64_t T, double *scores, uint64_t *counts, int32_t *topk,
                                     apo_corpus_report *report) {
	if (!e) return APO_E_ARG;
	if (!pc) return fail(e, APO_E_ARG, "input is NULL");
	HostTensor h{apo::CAND_Q, C, T, {{pc, 4}, {pd, 2}}, 2, true, codebook, d2book};
	return score_host(e, o, h, scores, counts, topk, report);
}

// =============================================================================== Form T (dictionary indices, 3 B / evaluation)
extern "C" int apo_score_host_tuples(apo_engine *e, const apo_score_opts *o, const uint16_t *tl, const uint8_t *th, const uint32_t *tbook_pc,
                                     const uint16_t *tbook_pd, uint32_t n_tuples, const uint32_t *codebook, const uint32_t *d2book,
                                     uint32_t C, uint64_t T, double *scores, uint64_t *counts, int32_t *topk, apo_corpus_report *report) {
	const HostTensor h{apo::CAND_T, C, T, {{tl, 2}, {th, 1}}, 2, false, codebook, d2book, tbook_pc, tbook_pd, n_tuples};
	return score_host(e, o, h, scores, counts, topk, report);
}

extern "C" int apo_tuples_upload(apo_engine *e, const uint16_t *tl, const uint8_t *th, const uint32_t *tbook_pc, const uint16_t *tbook_pd,
                                 uint32_t n_tuples, const uint32_t *codebook, const uint32_t *d2book, uint32_t C, uint64_t T) {
	if (!e) return APO_E_ARG;
	int rc;
	if ((rc = tuples_args(e, tl, th, tbook_pc, tbook_pd, n_tuples, codebook, d2book, C, T))) return rc;
	CK(cudaSetDevice(e->device));
	e->tup.unload();
	const uint64_t pitch = round_up(T ? T : 1, 64);                // rows start 16-byte aligned in both planes
	CK(reserve(e, e->tup.l, (uint64_t)C * pitch));
	CK(reserve(e, e->tup.h, (uint64_t)C * pitch));
	if ((rc = dict_upload(e, e->tup, tbook_pc, tbook_pd, n_tuples, codebook, d2book))) return rc;
	if ((rc = h2d_rows(e, e->tup.l.p, pitch * 2, tl, T * 2, T * 2, C, e->stream))) { cudaStreamSynchronize(e->stream); return rc; }
	if ((rc = h2d_rows(e, e->tup.h.p, pitch, th, T, T, C, e->stream))) { cudaStreamSynchronize(e->stream); return rc; }
	CK(cudaStreamSynchronize(e->stream));
	e->tup.C = C; e->tup.T = T; e->tup.pitch = pitch;
	return APO_OK;
}

namespace {
constexpr uint32_t kTwinTHot = 24576;   // K1t's shared-memory head of the table (KT_HOT_MAX, csrc/apo_tuple.cu)

template <class T>
int tb_reserve(apo_engine *e, DevBuf<T> &b, uint64_t n, const char *what, bool copy = false) {
	const cudaError_t c = copy ? b.reserve(n) : reserve(e, b, n);
	if (c == cudaSuccess) return APO_OK;
	cudaGetLastError();
	return fail(e, c == cudaErrorMemoryAllocation ? APO_E_NOMEM : APO_E_CUDA, "%s (%llu elements): %s", what, (unsigned long long)n, cudaGetErrorString(c));
}

void tb_release(apo_engine *e, int rc) {
	if (rc != APO_OK) cudaStreamSynchronize(e->stream);          // nothing a failed build queued may still use what is released
	e->tb_table.release(); e->tb_keys.release(); e->tb_cnt.release(); e->tb_misc.release();
}

// Form T of the loaded evaluations into D: the engine's resident Form T (apo_dims_tuples), or the Form T copy of its Form D
// tensor (copy, build_twin_t; *n_high: the evaluations whose index is >= 2^16).  The copy's buffers do not go through
// reserve: releasing the copies to make room would release the one being built.
int dims_tuples(apo_engine *e, uint32_t cap, uint32_t *n_tuples, TupleTensor &D, bool copy, uint64_t *n_high = nullptr) {
	if ((!e->dims_ptr && !e->compact) || e->dims_C == 0) return fail(e, APO_E_STATE, "no dims loaded");
	if (!e->compact && (!e->twin || e->env_no_twin))
		return fail(e, APO_E_STATE, "the loaded Form D tensor has no Form W / Q copy to build Form T from (APO_TUNE_NO_TWIN, apo_dims_attach, "
		                            "or too little device memory at load): call apo_dims_compact first");
	if (e->compact || !e->twin_w)
		for (int j = 0; j < 8; j++)
			if (e->qt.book[256 * j + 15] != 0xFFFFFFFFu)
				return fail(e, APO_E_STATE, "coded dimension %d takes 16 or more distinct values: Form T (like Form P) needs <= 15", j < 2 ? j : j + 1);
	if (cap > APO_TUPLES_MAX) cap = APO_TUPLES_MAX;
	const uint32_t C = e->dims_C;
	const uint64_t T = e->dims_T, pitch = e->dims_pitch, N = (uint64_t)C * T;
	const uint64_t m = std::min<uint64_t>(cap, N);                // at most this many dictionary entries
	uint64_t slots = 1024;
	while (slots < 2 * (m + 1)) slots <<= 1;
	const uint64_t tpitch = round_up(T ? T : 1, 64);               // as apo_tuples_upload
	// everything is allocated before the source is chosen: reserve may release the copy this build reads
	int rc;
	if ((rc = tb_reserve(e, D.l, (uint64_t)C * tpitch, "Form T low plane", copy)) || (rc = tb_reserve(e, D.h, (uint64_t)C * tpitch, "Form T high plane", copy)) ||
	    (rc = tb_reserve(e, D.pc, m ? m : 1, "dictionary", copy)) || (rc = tb_reserve(e, D.pd, m ? m : 1, "dictionary", copy)) ||
	    (rc = tb_reserve(e, D.d2, 4096, "d2book", copy)) || (rc = tb_reserve(e, e->tb_table, 2 * slots, "hash table", copy)) ||
	    (rc = tb_reserve(e, e->tb_keys, m ? m : 1, "keys", copy)) || (rc = tb_reserve(e, e->tb_cnt, m ? m : 1, "counts", copy)) ||
	    (rc = tb_reserve(e, e->tb_misc, 4, "counters", copy)))
		return rc;
	if (!e->compact && !e->twin)
		return fail(e, APO_E_NOMEM, "device memory ran short: the Form W / Q copy of the loaded tensor was released to make room for the build; "
		                            "free device memory and load the tensor again, or call apo_dims_compact");
	apo::TbSource S{};
	if (e->twin_w && !e->compact) S.qw = e->qw.p;
	else { S.q8 = e->q8.p; S.d2 = e->qd2.p; S.li = e->qli.p; }
	S.pitch = pitch; S.C = C; S.T = T;
	unsigned long long *misc = e->tb_misc.p;                       // [0] keys inserted, [1] over flag / index miss, [2] compacted
	CK(cudaMemsetAsync(misc, 0, 4 * 8, e->stream));
	uint32_t n = 0;
	std::vector<unsigned long long> keys, counts;
	if (N) {
		CK(apo::run_tb_clear(e->tb_table.p, slots, e->stream));
		CK(apo::run_tb_count(S, e->tb_table.p, slots, cap, misc, (uint32_t *)(misc + 1), e->sm_count, e->stream));
		unsigned long long h[2];
		CK(cudaMemcpyAsync(h, misc, sizeof h, cudaMemcpyDeviceToHost, e->stream));
		CK(cudaStreamSynchronize(e->stream));
		if (h[1]) {
			*n_tuples = h[0] > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)h[0];
			return fail(e, APO_E_STATE, "the evaluations hold more than cap=%u distinct ones (at least %llu): keep Form W / Q", cap, h[0]);
		}
		n = (uint32_t)h[0];
		CK(apo::run_tb_compact(e->tb_table.p, slots, e->tb_keys.p, e->tb_cnt.p, misc + 2, e->stream));
		keys.resize(n); counts.resize(n);
		CK(cudaMemcpyAsync(keys.data(), e->tb_keys.p, (uint64_t)n * 8, cudaMemcpyDeviceToHost, e->stream));
		CK(cudaMemcpyAsync(counts.data(), e->tb_cnt.p, (uint64_t)n * 8, cudaMemcpyDeviceToHost, e->stream));
		CK(cudaStreamSynchronize(e->stream));
	}
	// d2book: the distinct tool_success_rate values in ensure_d2book's order; a key's high half becomes its index
	std::vector<uint32_t> d2;
	for (uint32_t i = 0; i < n; i++) if ((uint32_t)(keys[i] >> 32) != apo::KW_D2_ABSENT) d2.push_back((uint32_t)(keys[i] >> 32));
	std::sort(d2.begin(), d2.end());
	d2.erase(std::unique(d2.begin(), d2.end()), d2.end());
	if (d2.size() > 4095) return fail(e, APO_E_STATE, "tool_success_rate takes %zu distinct values: more than the 4095 Form T can index", d2.size());
	std::sort(d2.begin(), d2.end(), d2_before);
	uint32_t d2book[4096];
	for (size_t c = 0; c < 4096; c++) d2book[c] = c < d2.size() ? d2[c] : 0xFFFFFFFFu;
	// dictionary order: count desc, then tuple_key (code word | d2book index << 32) asc, as apo_tuple_encode_host
	std::vector<std::pair<unsigned long long, unsigned long long>> order(n);     // (count, tuple key)
	for (uint32_t i = 0; i < n; i++) {
		const uint32_t hi = (uint32_t)(keys[i] >> 32);
		const uint64_t pd = hi == apo::KW_D2_ABSENT ? 4095u : (uint64_t)(std::lower_bound(d2.begin(), d2.end(), hi, d2_before) - d2.begin());
		order[i] = {counts[i], (keys[i] & 0xFFFFFFFFull) | (pd << 32)};
	}
	std::sort(order.begin(), order.end(), [](const std::pair<unsigned long long, unsigned long long> &x, const std::pair<unsigned long long, unsigned long long> &y) {
		if (x.first != y.first) return x.first > y.first;
		return x.second < y.second;
	});
	if (copy) {                                                   // see build_twin_t
		uint64_t head = 0;
		for (uint32_t r = 0; r < n && r < kTwinTHot; r++) head += order[r].first;
		if (head * 4 < N * 3) return APO_E_STATE;
		*n_high = 0;
		for (uint32_t r = 65536; r < n; r++) *n_high += order[r].first;
	}
	std::vector<uint32_t> tb_pc(n);
	std::vector<uint16_t> tb_pd(n);
	for (uint32_t r = 0; r < n; r++) {
		const uint32_t pd = (uint32_t)(order[r].second >> 32);
		tb_pc[r] = (uint32_t)order[r].second; tb_pd[r] = (uint16_t)pd;
		keys[r] = (unsigned long long)tb_pc[r] | ((unsigned long long)(pd == 4095u ? apo::KW_D2_ABSENT : d2book[pd]) << 32);   // back to the evaluation key
	}
	CK(cudaMemcpyAsync(D.d2.p, d2book, sizeof d2book, cudaMemcpyHostToDevice, e->stream));
	if (n) {
		CK(cudaMemcpyAsync(D.pc.p, tb_pc.data(), (uint64_t)n * 4, cudaMemcpyHostToDevice, e->stream));
		CK(cudaMemcpyAsync(D.pd.p, tb_pd.data(), (uint64_t)n * 2, cudaMemcpyHostToDevice, e->stream));
		CK(cudaMemcpyAsync(e->tb_keys.p, keys.data(), (uint64_t)n * 8, cudaMemcpyHostToDevice, e->stream));
		// the index table holds only the dictionary (slots >= 2 n, so that it stays small enough for L2)
		uint64_t islots = 1024;
		while (islots < 2ull * n) islots <<= 1;
		CK(apo::run_tb_clear(e->tb_table.p, islots, e->stream));
		CK(apo::run_tb_insert(e->tb_keys.p, n, e->tb_table.p, islots, e->stream));
		CK(apo::run_tb_index(S, e->tb_keys.p, n, e->tb_table.p, islots, D.l.p, D.h.p, tpitch, (uint32_t *)(misc + 1), e->sm_count, e->stream));
	}
	unsigned long long miss = 0;
	CK(cudaMemcpyAsync(&miss, misc + 1, 8, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	if (miss) return fail(e, APO_E_CUDA, "internal error: an evaluation's key is missing from the dictionary");
	memcpy(D.book, e->qt.book, sizeof D.book);
	D.C = C; D.T = T; D.pitch = tpitch; D.n = n;
	*n_tuples = n;
	return APO_OK;
}

// The Form T copy of a freshly loaded Form D tensor that holds a Form W / Q copy with <= 15 values per coded dimension: its
// resident Form D calls then read 3 B per evaluation through K1t (route_twin).  Built when the tensor holds at least
// kTwinTMinEvals evaluations (APO_TUNE_TWIN_T: any size), at most kTwinTCap distinct ones (the build's scratch is sized
// from it; the table stays well inside L2), the kTwinTHot most frequent of them cover at least 3/4 of the evaluations (K1t
// serves those from shared memory and gathers the rest from L2: on an H100 it beats K1q on Form W with 75 % of its reads in
// the head and loses by 2x with 9 %, DESIGN §8), and kTwinHeadroom of device memory stays free beside the copy and the
// build's scratch; otherwise no copy is kept, without an error.  The build also computes the table values for the weights.
constexpr uint64_t kTwinTMinEvals = 1ull << 26;
constexpr uint32_t kTwinTCap = 1u << 20;

// The exception list of the Form T copy: with it resident Form D calls read 2 B per evaluation through K1t2 instead of 3 B
// through K1t (route_twin).  Built from n_high, the evaluations whose index is >= 2^16 (known from the dictionary's
// counts), when at most 1/kTwinT2Share of the evaluations are such exceptions (DESIGN §8: K1t2 corrects each one with
// three dependent loads after its stream) and a row's positions fit 32 bits; otherwise, or without room for it, the copy
// is read through K1t as before, without an error.  APO_TUNE_NO_TWIN_T2 at the load builds none.
constexpr uint64_t kTwinT2Share = 64;
int build_twin_t2(apo_engine *e, uint64_t n_high) {
	TupleCopy &t = e->tcopy;
	const uint32_t C = t.C;
	const uint64_t T = t.T;
	if (e->env_no_twin_t2 || n_high * kTwinT2Share > (uint64_t)C * T || T > 0xFFFFFFFFull || n_high > 0xFFFFFFFFull) return APO_OK;
	if (n_high) {
		const uint32_t nblk = (uint32_t)((T + apo::KT_XBLOCK - 1) / apo::KT_XBLOCK);
		if (t.xb.reserve((uint64_t)C * (nblk + 1)) != cudaSuccess || t.xs.reserve(n_high) != cudaSuccess) {
			cudaGetLastError();
			t.xb.release(); t.xs.release();
			return APO_OK;
		}
		CK(apo::run_tx_build(t.l.p, t.h.p, t.pitch, C, T, t.xb.p, t.xs.p, e->sm_count, e->stream));
		CK(cudaStreamSynchronize(e->stream));                     // the load returns with the list built, as with the copy
		t.xn = n_high; t.nblk = nblk;
	}
	t.t2 = true;
	return APO_OK;
}

int build_twin_t(apo_engine *e) {
	const uint32_t C = e->dims_C;
	const uint64_t T = e->dims_T, N = (uint64_t)C * T;
	if (e->env_no_twin_t || !(N >= kTwinTMinEvals || e->env_twin_t)) return APO_OK;
	if (!e->twin_w)
		for (int j = 0; j < 8; j++)
			if (e->qt.book[256 * j + 15] != 0xFFFFFFFFu) return APO_OK;
	const uint64_t m = std::min<uint64_t>(kTwinTCap, N);
	uint64_t slots = 1024;
	while (slots < 2 * (m + 1)) slots <<= 1;
	// index planes, dictionary, value tables, the largest exception list and its block index; the build's hash table, keys
	// and counts
	const uint64_t need = 3 * (uint64_t)C * round_up(T, 64) + m * 6 + 2 * (m + 1) * 8 + 8 * (N / kTwinT2Share) +
	                      4 * (uint64_t)C * (T / apo::KT_XBLOCK + 2) + 16 * slots + 16 * m;
	size_t free_bytes = 0, total_bytes = 0;
	CK(cudaMemGetInfo(&free_bytes, &total_bytes));
	if ((uint64_t)free_bytes < need + kTwinHeadroom) return APO_OK;
	const std::string keep_err = e->err;
	uint32_t n = 0;
	uint64_t n_high = 0;
	TupleVals &v = e->tcopy.vals;
	int rc = dims_tuples(e, kTwinTCap, &n, e->tcopy, true, &n_high);
	if (rc == APO_OK && (v.val[0].reserve(n + 1ull) != cudaSuccess || v.val[1].reserve(n + 1ull) != cudaSuccess ||
	                     v.ptab.reserve(8 * 256) != cudaSuccess || v.bad.reserve(1) != cudaSuccess)) {
		cudaGetLastError();
		rc = APO_E_NOMEM;
	}
	if (rc == APO_OK) rc = tuple_values(e, e->tcopy, v, false);
	if (rc == APO_OK) rc = build_twin_t2(e, n_high);
	tb_release(e, rc);
	if (rc == APO_OK) return APO_OK;
	e->tcopy.release();
	if (rc != APO_E_STATE && rc != APO_E_NOMEM) return rc;
	e->err = keep_err;                                          // more than kTwinTCap distinct evaluations, or no room: no copy
	return APO_OK;
}
}  // namespace

extern "C" int apo_dims_tuples(apo_engine *e, uint32_t cap, uint32_t *n_tuples) {
	if (!e) return APO_E_ARG;
	if (!n_tuples) return fail(e, APO_E_ARG, "n_tuples is NULL");
	*n_tuples = 0;
	CK(cudaSetDevice(e->device));
	e->tup.unload();                                               // a failure leaves no Form T loaded, as a failed apo_tuples_upload
	const int rc = dims_tuples(e, cap, n_tuples, e->tup, false);
	tb_release(e, rc);
	return rc;
}

extern "C" int apo_tuples_download(apo_engine *e, uint16_t *tl, uint8_t *th, uint32_t c, uint64_t first, uint64_t n) {
	if (!e || !tl || !th) return fail(e, APO_E_ARG, "NULL argument");
	if (e->tup.l.p == nullptr || e->tup.C == 0) return fail(e, APO_E_STATE, "no tuples loaded");
	if (c >= e->tup.C || first > e->tup.T || n > e->tup.T - first) return fail(e, APO_E_ARG, "range outside the tuples");
	if (n == 0) return APO_OK;
	CK(cudaSetDevice(e->device));
	const uint64_t off = (uint64_t)c * e->tup.pitch + first;
	CK(cudaMemcpyAsync(tl, e->tup.l.p + off, n * 2, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaMemcpyAsync(th, e->tup.h.p + off, n, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	return APO_OK;
}

extern "C" int apo_tuples_book(apo_engine *e, uint32_t *tbook_pc, uint16_t *tbook_pd, uint32_t cap, uint32_t *codebook, uint32_t *d2book,
                               uint32_t *n_tuples) {
	if (!e || !n_tuples) return fail(e, APO_E_ARG, "NULL argument");
	if (e->tup.l.p == nullptr || e->tup.C == 0) return fail(e, APO_E_STATE, "no tuples loaded");
	const uint32_t n = e->tup.n;
	*n_tuples = n;
	if (cap < n) return fail(e, APO_E_ARG, "cap=%u is smaller than the %u dictionary entries", cap, n);
	if (!codebook || !d2book || (n && (!tbook_pc || !tbook_pd))) return fail(e, APO_E_ARG, "NULL argument");
	CK(cudaSetDevice(e->device));
	if (n) {
		CK(cudaMemcpyAsync(tbook_pc, e->tup.pc.p, (uint64_t)n * 4, cudaMemcpyDeviceToHost, e->stream));
		CK(cudaMemcpyAsync(tbook_pd, e->tup.pd.p, (uint64_t)n * 2, cudaMemcpyDeviceToHost, e->stream));
	}
	CK(cudaMemcpyAsync(d2book, e->tup.d2.p, 4096 * 4, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	memcpy(codebook, e->tup.book, sizeof e->tup.book);
	return APO_OK;
}

extern "C" int apo_host_alloc(uint64_t bytes, void **out) {
	if (!out) return APO_E_ARG;
	*out = nullptr;
	const cudaError_t c = cudaMallocHost(out, bytes ? bytes : 1);
	if (c != cudaSuccess) { cudaGetLastError(); return fail(nullptr, c == cudaErrorMemoryAllocation ? APO_E_NOMEM : APO_E_CUDA, "cudaMallocHost(%llu): %s", (unsigned long long)bytes, cudaGetErrorString(c)); }
	return APO_OK;
}

extern "C" int apo_host_free(void *p) {
	if (!p) return APO_OK;
	return cudaFreeHost(p) == cudaSuccess ? APO_OK : APO_E_CUDA;
}

extern "C" int apo_score_host(apo_engine *e, const apo_score_opts *o, const float *dims, uint32_t C, uint64_t T,
                              double *scores, uint64_t *counts, int32_t *topk, apo_corpus_report *report) {
	return score_host(e, o, {apo::CAND_DIMS, C, T, {{dims, 36}}, 1}, scores, counts, topk, report);
}

extern "C" int apo_score_host_records(apo_engine *e, const apo_score_opts *o, const void *recs, uint32_t row_bytes, uint32_t C, uint64_t T,
                                      double *scores, uint64_t *counts, int32_t *topk, apo_corpus_report *report) {
	if (row_bytes != 32 && row_bytes != 16) return fail(e, APO_E_ARG, "row_bytes must be 32 (apo_record) or 16 (apo_record16)");
	return score_host(e, o, {row_bytes == 32 ? apo::CAND_REC32 : apo::CAND_REC16, C, T, {{recs, row_bytes}}, 1}, scores, counts, topk, report);
}

extern "C" int apo_last_timing(const apo_engine *e, apo_timing *out) {
	if (!e || !out) return APO_E_ARG;
	*out = e->timing;
	return APO_OK;
}

extern "C" int apo_debug_partials(apo_engine *e, int64_t *out, uint32_t C) {
	if (!e || !out) return fail(e, APO_E_ARG, "NULL argument");
	if (C != e->last_C || !e->acc.p) return fail(e, APO_E_STATE, "no scoring call with C=%u to read back", C);
	CK(cudaSetDevice(e->device));
	CK(cudaMemcpyAsync(out, e->partials_src ? e->partials_src : e->acc.p, 8ull * ACC_PER_CAND * C, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	return APO_OK;
}

extern "C" int apo_debug_twin_t_list(apo_engine *e, uint64_t *n_words, uint64_t *n_exceptions, uint32_t *xb, uint32_t *xs) {
	if (!e || !n_words || !n_exceptions) return fail(e, APO_E_ARG, "NULL argument");
	*n_words = e->tcopy.xn ? (uint64_t)e->tcopy.C * (e->tcopy.nblk + 1) : 0;
	*n_exceptions = e->tcopy.xn;
	if (!e->tcopy.xn) return APO_OK;
	CK(cudaSetDevice(e->device));
	if (xb) CK(cudaMemcpyAsync(xb, e->tcopy.xb.p, *n_words * 4, cudaMemcpyDeviceToHost, e->stream));
	if (xs) CK(cudaMemcpyAsync(xs, e->tcopy.xs.p, e->tcopy.xn * 8, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	return APO_OK;
}

extern "C" int apo_candidate_reports(apo_engine *e, uint32_t c0, uint32_t n, apo_candidate_report *out) {
	if (!e) return APO_E_ARG;
	if (!e->cand_ready) return fail(e, APO_E_STATE, "the last scoring call did not set APO_SCORE_CANDIDATES");
	if ((uint64_t)c0 + n > e->cand_C) return fail(e, APO_E_ARG, "candidates [%u,%llu) exceed C=%u", c0, (unsigned long long)c0 + n, e->cand_C);
	if (n == 0) return APO_OK;
	if (!out) return fail(e, APO_E_ARG, "out is NULL");
	CK(cudaSetDevice(e->device));
	CK(cudaMemcpyAsync(out, e->cand_rep.p + c0, (uint64_t)n * sizeof(apo_candidate_report), cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	return APO_OK;
}

extern "C" int apo_candidate_corpus_reports(apo_engine *e, uint32_t c0, uint32_t n, apo_corpus_report *out) {
	if (!e) return APO_E_ARG;
	if (!e->ccorp_ready) return fail(e, APO_E_STATE, "the last scoring call did not set APO_SCORE_CANDIDATE_CORPUS");
	if ((uint64_t)c0 + n > e->ccorp_C) return fail(e, APO_E_ARG, "candidates [%u,%llu) exceed C=%u", c0, (unsigned long long)c0 + n, e->ccorp_C);
	if (n == 0) return APO_OK;
	if (!out) return fail(e, APO_E_ARG, "out is NULL");
	CK(cudaSetDevice(e->device));
	CK(cudaMemcpyAsync(out, e->ccorp_rep.p + c0, (uint64_t)n * sizeof(apo_corpus_report), cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	return APO_OK;
}

// =============================================================================== multi-GPU
extern "C" int apo_comm_unique_id(uint8_t out[APO_UNIQUE_ID_BYTES]) {
	if (!out) return fail(nullptr, APO_E_ARG, "out is NULL");
	std::string err;
	if (!nccl_load(err)) return fail(nullptr, APO_E_NCCL, "%s", err.c_str());
	NcclId id;
	const int rc = g_nccl.GetUniqueId(&id);
	if (rc != 0) return fail(nullptr, APO_E_NCCL, "ncclGetUniqueId failed (%d)", rc);
	memcpy(out, id.b, APO_UNIQUE_ID_BYTES);
	return APO_OK;
}

extern "C" int apo_comm_init(apo_engine *e, int nranks, int rank, const uint8_t id[APO_UNIQUE_ID_BYTES]) {
	if (!e || !id) return fail(e, APO_E_ARG, "NULL argument");
	if (nranks < 1 || rank < 0 || rank >= nranks) return fail(e, APO_E_ARG, "bad rank %d of %d", rank, nranks);
	CK(cudaSetDevice(e->device));
	peer_teardown(e);
	if (e->comm) { g_nccl.CommDestroy(e->comm); e->comm = nullptr; }
	e->nranks = 1; e->rank = 0;
	if (nranks == 1) return APO_OK;
	std::string err;
	if (!nccl_load(err)) return fail(e, APO_E_NCCL, "%s", err.c_str());
	NcclId nid; memcpy(nid.b, id, APO_UNIQUE_ID_BYTES);
	void *comm = nullptr;
	const int rc = g_nccl.CommInitRank(&comm, nranks, nid, rank);
	if (rc != 0) return fail(e, APO_E_NCCL, "ncclCommInitRank: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "error");
	e->comm = comm; e->nranks = nranks; e->rank = rank; e->acc_clean_words = 0; e->partials_src = nullptr;
	// one tiny allreduce now so that the first scoring call does not pay NCCL's lazy connection setup (~1 s)
	CK(reserve(e, e->misc, 32));
	CK(cudaMemsetAsync(e->misc.p + 24, 0, 8, e->stream));
	const int wrc = g_nccl.AllReduce(e->misc.p + 24, e->misc.p + 24, 1, kNcclInt64, kNcclSum, e->comm, e->stream);
	if (wrc != 0) return fail(e, APO_E_NCCL, "ncclAllReduce (warm-up): %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(wrc) : "error");
	CK(cudaStreamSynchronize(e->stream));
	// the join itself runs over NVLink peer memory inside the scoring launch; NCCL stays as the bootstrap and the fallback
	return peer_setup(e);
}

extern "C" int apo_comm_join_mode(const apo_engine *e) {
	if (!e || e->nranks <= 1) return 0;
	return (e->peer_ok && !e->env_nccl_join) ? 2 : 1;
}

extern "C" int apo_comm_destroy(apo_engine *e) {
	if (!e) return APO_E_ARG;
	cudaSetDevice(e->device);
	if (e->own_stream) cudaStreamSynchronize(e->stream);
	peer_teardown(e);
	if (e->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(e->comm);
	e->comm = nullptr; e->nranks = 1; e->rank = 0;
	return APO_OK;
}
