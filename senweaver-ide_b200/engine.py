"""ctypes binding of libapo_b200.so (include/apo_b200.h) — the host side of the C ABI.

This module is plumbing only: it loads the in-tree shared library, declares every entry
point of the header and wraps the engine handle in a small class that moves numpy buffers
across the boundary.  There is no CPU path here: if the library is missing or no H100 is
visible, construction raises (`ApoError`), it never falls back.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libapo_b200.so")

NDIM, NPAT, NMODE = 9, 6, 5
SRC_DIMS, SRC_ROLLOUTS, SRC_TUPLES = 0, 1, 2
TUPLES_MAX = 0xFFFFFF
SCORE_CORPUS, SCORE_RECIP, SCORE_TIMING, SCORE_CANDIDATES = 0x1, 0x2, 0x4, 0x8
SCORE_CANDIDATE_CORPUS = 0x10
SCORE_CANDIDATE_EXTREMES = 0x20
EXTREMES_N = 32
SCORE_CANDIDATE_GROUPS = 0x40
GROUPS_MAX = 64
SCORE_CANDIDATE_SPREAD = 0x80
SCORE_CANDIDATE_PAIRS = 0x100
SCORE_CANDIDATE_GROUP_PAIRS = 0x200
PAIR_NONE = 0xFFFFFFFF
TUNE_NO_FUSE, TUNE_FORCE_FUSE, TUNE_NO_STAGING, TUNE_NCCL_JOIN, TUNE_NO_TWIN = 0x1, 0x2, 0x4, 0x8, 0x10
TUNE_NO_TWIN_T, TUNE_TWIN_T, TUNE_NO_TWIN_T2, TUNE_NO_TWIN_H = 0x20, 0x40, 0x80, 0x100
TUNE_NO_CORPUS_DIGEST = 0x200
F_ERRORS, F_ENDED, F_VALID, F_FAILSPAN = 0x01, 0x02, 0x08, 0x10
UNIQUE_ID_BYTES = 128

DIM_NAMES = (
    "user_feedback", "task_completion", "tool_success_rate", "tool_call_reliability",
    "tool_call_efficiency", "tool_duration_efficiency", "response_efficiency",
    "token_efficiency", "conversation_efficiency",
)
MODE_NAMES = ("unknown", "normal", "agent", "gather", "designer")

RECORD_DTYPE = np.dtype([
    ("feedback", "u1"), ("flags", "u1"), ("mode", "u1"), ("durClass", "u1"),
    ("userMsgs", "<u2"), ("asstMsgs", "<u2"),
    ("toolCalls", "<u4"), ("toolSucc", "<u4"), ("toolFail", "<u4"),
    ("llmCalls", "<u4"), ("tokens", "<u4"), ("toolDurMs", "<f4"),
])
assert RECORD_DTYPE.itemsize == 32
RECORD16_DTYPE = np.dtype([
    ("hdr", "<u2"), ("userMsgs", "u1"), ("asstMsgs", "u1"), ("toolCalls", "<u2"), ("toolFail", "<u2"),
    ("llmCalls", "u1"), ("durClass", "u1"), ("tokens", "<u2"), ("toolDurMs", "<f4"),
])
assert RECORD16_DTYPE.itemsize == 16


class Pattern(C.Structure):
    _fields_ = [("count", C.c_uint64), ("flag", C.c_uint8), ("severity", C.c_uint8), ("pad", C.c_uint8 * 6),
                ("examples", C.c_int64 * 3)]


class DimStat(C.Structure):
    _fields_ = [("sum", C.c_double), ("count", C.c_uint64), ("avg", C.c_double),
                ("low_flag", C.c_uint8), ("low_severity", C.c_uint8), ("sugg_flag", C.c_uint8),
                ("sugg_priority", C.c_uint8), ("pad", C.c_uint8 * 4)]


class CorpusReport(C.Structure):
    _fields_ = [("total", C.c_uint64), ("good", C.c_uint64), ("bad", C.c_uint64), ("none", C.c_uint64),
                ("goodRate", C.c_double), ("byMode", (C.c_uint64 * 3) * NMODE), ("byModeGoodRate", C.c_double * NMODE),
                ("withReward", C.c_uint64), ("rewardSum", C.c_double), ("avgReward", C.c_double),
                ("dim", DimStat * NDIM), ("pat", Pattern * NPAT),
                ("toolCalls", C.c_uint64), ("toolSucc", C.c_uint64), ("toolFail", C.c_uint64),
                ("toolSuccessRate", C.c_double)]


class CandidateReport(C.Structure):
    """apo_candidate_report: the corpus report's numbers for one candidate over the evaluations a call scored."""
    _fields_ = [("total", C.c_uint64), ("good", C.c_uint64), ("bad", C.c_uint64), ("none", C.c_uint64),
                ("goodRate", C.c_double), ("withReward", C.c_uint64), ("rewardSum", C.c_double), ("avgReward", C.c_double),
                ("dim", DimStat * NDIM), ("badExamples", C.c_int64 * 3)]


class CandidateExtremes(C.Structure):
    """struct apo_candidate_extremes: the EXTREMES_N lowest- and highest-reward evaluations of one candidate (record positions,
    -1 / NaN past n)."""
    _fields_ = [("n", C.c_uint64), ("lowest", C.c_int64 * EXTREMES_N), ("lowestReward", C.c_double * EXTREMES_N),
                ("highest", C.c_int64 * EXTREMES_N), ("highestReward", C.c_double * EXTREMES_N)]


class GroupScore(C.Structure):
    """apo_group_score: candidate c's evaluations on the records of one group (tallies, non-null count, exact reward sum and
    mean; avgReward NaN when withReward == 0)."""
    _fields_ = [("total", C.c_uint64), ("good", C.c_uint64), ("bad", C.c_uint64), ("goodRate", C.c_double),
                ("withReward", C.c_uint64), ("rewardSum", C.c_double), ("avgReward", C.c_double)]


class CandidateSpread(C.Structure):
    """struct apo_candidate_spread: one candidate's reward spread.  n == counts[c]; the exact integers S1 = sum x (two's
    complement 128-bit: sumLo, sumHi) and S2 = sum x^2 (unsigned 192-bit, sumSq least significant word first) of its terms
    x = rint(fr * 2^52); mean == scores[c] (NaN when n == 0); rewardSumSq = RN(S2) * 2^-104; the unbiased variance, stdDev
    and stdErr of the mean, each rounded as the header states (NaN when n < 2)."""
    _fields_ = [("n", C.c_uint64), ("sumLo", C.c_uint64), ("sumHi", C.c_int64), ("sumSq", C.c_uint64 * 3),
                ("mean", C.c_double), ("rewardSumSq", C.c_double), ("variance", C.c_double), ("stdDev", C.c_double),
                ("stdErr", C.c_double)]

    @property
    def sum(self) -> int:
        """S1 as a Python int"""
        return (int(self.sumHi) << 64) | int(self.sumLo)

    @property
    def sum_sq(self) -> int:
        """S2 as a Python int"""
        return int(self.sumSq[0]) | (int(self.sumSq[1]) << 64) | (int(self.sumSq[2]) << 128)


class CandidatePair(C.Structure):
    """struct apo_candidate_pair: one candidate compared with its reference on the record positions both were scored on.
    ref (PAIR_NONE: no reference, every count 0, every double NaN); n positions where both have a finalReward, with wins /
    losses / ties as d = x_c - x_r > 0 / < 0 / == 0 of the terms x = rint(fr * 2^52); candOnly / refOnly positions where only
    one of them has a finalReward (left out of the sums); the exact integers D1 = sum d (two's complement 128-bit: sumLo,
    sumHi) and D2 = sum d^2 (unsigned 192-bit, sumSq least significant word first); meanDiff (NaN when n == 0), the unbiased
    variance, stdDev and stdErr of the paired differences, each rounded as the header states (NaN when n < 2)."""
    _fields_ = [("ref", C.c_uint32), ("pad", C.c_uint32), ("n", C.c_uint64), ("wins", C.c_uint64), ("losses", C.c_uint64),
                ("ties", C.c_uint64), ("candOnly", C.c_uint64), ("refOnly", C.c_uint64), ("sumLo", C.c_uint64), ("sumHi", C.c_int64),
                ("sumSq", C.c_uint64 * 3), ("meanDiff", C.c_double), ("variance", C.c_double), ("stdDev", C.c_double),
                ("stdErr", C.c_double)]

    @property
    def sum(self) -> int:
        """D1 as a Python int"""
        return (int(self.sumHi) << 64) | int(self.sumLo)

    @property
    def sum_sq(self) -> int:
        """D2 as a Python int"""
        return int(self.sumSq[0]) | (int(self.sumSq[1]) << 64) | (int(self.sumSq[2]) << 128)


class Timing(C.Structure):
    _fields_ = [("reward_ms", C.c_float), ("corpus_ms", C.c_float), ("allreduce_ms", C.c_float),
                ("finalize_ms", C.c_float), ("total_ms", C.c_float), ("launches", C.c_uint32), ("pad", C.c_uint32),
                ("join_wait_ms", C.c_float), ("join_reduce_ms", C.c_float), ("tail_finalize_ms", C.c_float), ("tail_publish_ms", C.c_float)]


class ScoreOpts(C.Structure):
    _fields_ = [("K", C.c_uint32), ("source", C.c_uint32), ("flags", C.c_uint32), ("variant", C.c_uint32),
                ("first", C.c_uint64), ("count", C.c_uint64)]


class ApoError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"apo_b200 error {code}: {msg}")
        self.code = code


# every symbol include/apo_b200.h declares (tests/test_abi_symbols.py checks the .so against this list)
ABI_SYMBOLS = (
    "apo_abi_version", "apo_create", "apo_destroy", "apo_last_error", "apo_set_stream", "apo_set_weights", "apo_set_tuning",
    "apo_get_weights", "apo_reward_batch", "apo_reward_one", "apo_corpus_upload", "apo_corpus_generate",
    "apo_corpus_download", "apo_records_from_json", "apo_corpus_upload_json", "apo_dims_upload", "apo_dims_generate", "apo_dims_download", "apo_dims_attach",
    "apo_dims_compact", "apo_dims_generate_compact", "apo_dims_upload_compact", "apo_dims_layout",
    "apo_rollouts_upload", "apo_rollouts_generate", "apo_rollouts_download", "apo_rollouts16_upload",
    "apo_rollouts16_generate", "apo_rollouts16_download", "apo_record_pack16", "apo_record_unpack16", "apo_duration_class", "apo_score",
    "apo_score_begin", "apo_score_accumulate", "apo_score_finish", "apo_score_host", "apo_score_host_records", "apo_score_host_compact", "apo_compact_encode_host",
    "apo_dims_compact_download", "apo_dims_codebook", "apo_packed_encode_host", "apo_score_host_packed", "apo_dims_packed_download", "apo_dims_d2book",
    "apo_tuple_encode_host", "apo_score_host_tuples", "apo_tuples_upload", "apo_dims_tuples", "apo_tuples_download", "apo_tuples_book",
    "apo_host_alloc", "apo_host_free",
    "apo_last_timing", "apo_debug_partials", "apo_debug_twin_t_list", "apo_debug_twin_h", "apo_debug_corpus_digest", "apo_candidate_reports", "apo_candidate_corpus_reports", "apo_candidate_extremes", "apo_record_groups_upload", "apo_candidate_groups", "apo_candidate_spread", "apo_candidate_refs_upload", "apo_candidate_pairs", "apo_candidate_group_pairs", "apo_comm_unique_id", "apo_comm_init", "apo_comm_destroy", "apo_comm_join_mode",
)


def build_library(force: bool = False) -> str:
    """Compile csrc/ for sm_90a in-tree (nvcc cross-compiles without a GPU)."""
    csrc = os.path.join(_HERE, "csrc")
    srcs = [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cu", ".cuh", ".h", ".cpp")) or f == "Makefile"]
    srcs.append(os.path.join(_HERE, "..", "include", "apo_b200.h"))
    stale = (not os.path.exists(LIB_PATH)) or any(os.path.getmtime(s) > os.path.getmtime(LIB_PATH) for s in srcs)
    if force or stale:
        r = subprocess.run(["make", "-s", "-C", csrc], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc build failed:\n" + r.stdout[-2000:] + r.stderr[-4000:])
    return LIB_PATH


_lib = None


def load_library() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        try:                                    # fresh checkout: compile the sm_90a library in-tree (nvcc needs no GPU)
            build_library()
        except Exception as ex:
            raise ApoError(-2, f"{LIB_PATH} is missing and could not be built ({ex}); run "
                               "`python -c 'import __graft_entry__ as g; g.build()'` (there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
    L.apo_abi_version.restype = i32
    L.apo_create.argtypes = [i32, C.POINTER(vp)]
    L.apo_destroy.argtypes = [vp]
    L.apo_destroy.restype = None
    L.apo_last_error.argtypes = [vp]
    L.apo_last_error.restype = C.c_char_p
    L.apo_set_stream.argtypes = [vp, u64]
    L.apo_set_weights.argtypes = [vp, vp]
    L.apo_set_tuning.argtypes = [vp, u32]
    L.apo_get_weights.argtypes = [vp, vp]
    L.apo_reward_batch.argtypes = [vp, vp, u64, vp, vp, vp]
    L.apo_reward_one.argtypes = [vp, vp, vp, vp, vp]
    L.apo_corpus_upload.argtypes = [vp, vp, u64, u64]
    L.apo_corpus_generate.argtypes = [vp, u64, u64, u64, u32]
    L.apo_corpus_download.argtypes = [vp, vp, u64, u64]
    L.apo_dims_upload.argtypes = [vp, vp, u32, u64]
    L.apo_dims_generate.argtypes = [vp, u64, u32, u32, u64, u64, u32]
    L.apo_dims_download.argtypes = [vp, vp, u32, u64, u64]
    L.apo_dims_attach.argtypes = [vp, u64, u32, u64, u64]
    L.apo_dims_compact.argtypes = [vp]
    L.apo_dims_generate_compact.argtypes = [vp, u64, u32, u32, u64, u64, u32]
    L.apo_dims_upload_compact.argtypes = [vp, vp, u32, u64]
    L.apo_dims_layout.argtypes = [vp]
    L.apo_rollouts_upload.argtypes = [vp, vp, u32, u64]
    L.apo_rollouts_generate.argtypes = [vp, u64, u32, u32, u64, u64, u32]
    L.apo_rollouts_download.argtypes = [vp, vp, u32, u64, u64]
    L.apo_rollouts16_upload.argtypes = [vp, vp, u32, u64]
    L.apo_rollouts16_generate.argtypes = [vp, u64, u32, u32, u64, u64, u32]
    L.apo_rollouts16_download.argtypes = [vp, vp, u32, u64, u64]
    L.apo_record_pack16.argtypes = [vp, u64, vp, vp]
    L.apo_record_unpack16.argtypes = [vp, u64, vp]
    L.apo_score_host_records.argtypes = [vp, C.POINTER(ScoreOpts), vp, u32, u32, u64, vp, vp, vp, vp]
    L.apo_score.argtypes = [vp, C.POINTER(ScoreOpts), vp, vp, vp, vp]
    L.apo_score_begin.argtypes = [vp, u32]
    L.apo_score_accumulate.argtypes = [vp, C.POINTER(ScoreOpts), u32]
    L.apo_score_finish.argtypes = [vp, C.POINTER(ScoreOpts), vp, vp, vp, vp]
    L.apo_score_host.argtypes = [vp, C.POINTER(ScoreOpts), vp, u32, u64, vp, vp, vp, vp]
    L.apo_score_host_compact.argtypes = [vp, C.POINTER(ScoreOpts), vp, vp, vp, vp, u32, u64, vp, vp, vp, vp]
    L.apo_compact_encode_host.argtypes = [vp, u32, u64, vp, vp, vp, vp, i32]
    L.apo_packed_encode_host.argtypes = [vp, u32, u64, vp, vp, vp, vp, i32]
    L.apo_dims_packed_download.argtypes = [vp, vp, vp, u32, u64, u64]
    L.apo_dims_d2book.argtypes = [vp, vp]
    L.apo_score_host_packed.argtypes = [vp, C.POINTER(ScoreOpts), vp, vp, vp, vp, u32, u64, vp, vp, vp, vp]
    L.apo_tuple_encode_host.argtypes = [vp, vp, u32, u64, vp, vp, vp, vp, u32, vp, i32]
    L.apo_score_host_tuples.argtypes = [vp, C.POINTER(ScoreOpts), vp, vp, vp, vp, u32, vp, vp, u32, u64, vp, vp, vp, vp]
    L.apo_tuples_upload.argtypes = [vp, vp, vp, vp, vp, u32, vp, vp, u32, u64]
    L.apo_dims_tuples.argtypes = [vp, u32, vp]
    L.apo_tuples_download.argtypes = [vp, vp, vp, u32, u64, u64]
    L.apo_tuples_book.argtypes = [vp, vp, vp, u32, vp, vp, vp]
    L.apo_dims_compact_download.argtypes = [vp, vp, vp, vp, u32, u64, u64]
    L.apo_dims_codebook.argtypes = [vp, vp]
    L.apo_last_timing.argtypes = [vp, C.POINTER(Timing)]
    L.apo_debug_partials.argtypes = [vp, vp, u32]
    L.apo_debug_twin_t_list.argtypes = [vp, vp, vp, vp, vp]
    L.apo_debug_twin_h.argtypes = [vp, vp, vp, vp, vp]
    L.apo_debug_corpus_digest.argtypes = [vp, vp, vp, vp]
    L.apo_candidate_reports.argtypes = [vp, u32, u32, vp]
    L.apo_candidate_corpus_reports.argtypes = [vp, u32, u32, vp]
    L.apo_candidate_extremes.argtypes = [vp, u32, u32, vp]
    L.apo_record_groups_upload.argtypes = [vp, vp, u64, u32]
    L.apo_candidate_groups.argtypes = [vp, u32, u32, u32, vp]
    L.apo_candidate_spread.argtypes = [vp, u32, u32, vp]
    L.apo_candidate_refs_upload.argtypes = [vp, vp, u32]
    L.apo_candidate_pairs.argtypes = [vp, u32, u32, vp]
    L.apo_candidate_group_pairs.argtypes = [vp, u32, u32, u32, vp]
    L.apo_comm_unique_id.argtypes = [vp]
    L.apo_comm_init.argtypes = [vp, i32, i32, vp]
    L.apo_comm_destroy.argtypes = [vp]
    L.apo_comm_join_mode.argtypes = [vp]
    for name in ABI_SYMBOLS:
        f = getattr(L, name)
        if name not in ("apo_destroy", "apo_last_error", "apo_records_from_json", "apo_duration_class"):
            f.restype = i32
    L.apo_duration_class.argtypes = [C.c_double, u32]
    L.apo_duration_class.restype = C.c_uint8
    L.apo_host_alloc.argtypes = [u64, C.POINTER(vp)]
    L.apo_host_free.argtypes = [vp]
    L.apo_records_from_json.argtypes = [C.c_char_p, u64, vp, u64, C.POINTER(u64)]
    L.apo_records_from_json.restype = C.c_int64
    L.apo_corpus_upload_json.argtypes = [vp, C.c_char_p, u64, u64, C.POINTER(u64)]
    _lib = L
    return L


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class _Pinned:
    """Owner of one apo_host_alloc block.  numpy arrays made from it (array interface) hold it as their base,
    so the block is released when the last view goes away."""

    def __init__(self, nbytes):
        self._L, self.ptr, self.nbytes = load_library(), C.c_void_p(), int(nbytes)
        rc = self._L.apo_host_alloc(self.nbytes, C.byref(self.ptr))
        if rc != 0:
            raise ApoError(rc, (self._L.apo_last_error(None) or b"").decode())

    @property
    def __array_interface__(self):
        return {"shape": (self.nbytes,), "typestr": "|u1", "data": (self.ptr.value, False), "version": 3}

    def __del__(self):
        if getattr(self, "ptr", None) is not None and self.ptr.value:
            self._L.apo_host_free(self.ptr)
            self.ptr = C.c_void_p()


def host_empty(shape, dtype) -> np.ndarray:
    """Page-locked host array (apo_host_alloc): the streaming calls read it in place at PCIe line rate."""
    dt = np.dtype(dtype)
    n = int(np.prod(shape)) * dt.itemsize
    return np.asarray(_Pinned(n)).view(dt).reshape(shape)


def records_from_json(text: str | bytes) -> np.ndarray:
    """apo_records_from_json: the reference's persisted trace array (TCS:296-359) -> Form R.  Host-side
    format code of the C library; needs no GPU.  Raises ValueError with the byte offset on malformed input."""
    L = load_library()
    raw = text.encode() if isinstance(text, str) else text
    pos = C.c_uint64(0)
    n = L.apo_records_from_json(raw, len(raw), None, 0, C.byref(pos))
    if n < 0:
        raise ValueError(f"malformed trace JSON at byte {pos.value}")
    out = np.zeros(n, RECORD_DTYPE)
    if n:
        L.apo_records_from_json(raw, len(raw), _p(out), n, C.byref(pos))
    return out


class ScoreResult:
    __slots__ = ("scores", "counts", "topk", "report", "timing", "candidates", "candidate_corpus", "extremes", "groups", "spread", "pairs", "group_pairs")

    def __init__(self, scores, counts, topk, report, timing, candidates=None, candidate_corpus=None, extremes=None, groups=None,
                 spread=None, pairs=None, group_pairs=None):
        self.scores, self.counts, self.topk, self.report, self.timing = scores, counts, topk, report, timing
        self.candidates = candidates        # CandidateReport array [C] when the call asked for the breakdown, else None
        self.candidate_corpus = candidate_corpus   # CorpusReport array [C] when the call asked for the per-candidate corpus reports
        self.extremes = extremes            # CandidateExtremes array [C] when the call asked for the per-candidate extremes
        self.groups = groups                # GroupScore array [C][G] when the call asked for the per-candidate group scores
        self.spread = spread                # CandidateSpread array [C] when the call asked for the per-candidate reward spread
        self.pairs = pairs                  # CandidatePair array [C] when the call asked for the paired comparisons
        self.group_pairs = group_pairs      # CandidatePair array [C][G] when the call asked for the per-group paired comparisons


class Engine:
    """One GPU, one handle.  Mirrors the C ABI one to one."""

    def __init__(self, device: int = 0):
        self._L = load_library()
        h = C.c_void_p()
        rc = self._L.apo_create(device, C.byref(h))
        if rc != 0:
            raise ApoError(rc, (self._L.apo_last_error(None) or b"").decode())
        self._h = h
        self.device = device
        self._groups_G = 0                  # G of the record groups held (record_groups_upload)

    # -- plumbing
    def close(self):
        if getattr(self, "_h", None):
            self._L.apo_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc: int):
        if rc != 0:
            raise ApoError(rc, (self._L.apo_last_error(self._h) or b"").decode())

    def set_stream(self, cuda_stream: int):
        self._ck(self._L.apo_set_stream(self._h, cuda_stream))

    def set_tuning(self, flags: int):
        """TUNE_* switches (experiments / tests); results are identical for every setting."""
        self._ck(self._L.apo_set_tuning(self._h, flags))

    def set_weights(self, w):
        w = np.ascontiguousarray(w, np.float64)
        assert w.shape == (NDIM,)
        self._ck(self._L.apo_set_weights(self._h, _p(w)))

    def get_weights(self) -> np.ndarray:
        w = np.empty(NDIM, np.float64)
        self._ck(self._L.apo_get_weights(self._h, _p(w)))
        return w

    # -- single-trace path (TCS:668-788)
    def reward_batch(self, recs: np.ndarray):
        recs = np.ascontiguousarray(recs, RECORD_DTYPE).reshape(-1)
        n = recs.shape[0]
        dims = np.empty((n, NDIM), np.float64)
        masks = np.empty(n, np.uint32)
        finals = np.empty(n, np.float64)
        self._ck(self._L.apo_reward_batch(self._h, _p(recs), n, _p(dims), _p(masks), _p(finals)))
        return dims, masks, finals

    # -- corpus
    def corpus_upload(self, recs: np.ndarray, idx_base: int = 0):
        recs = np.ascontiguousarray(recs, RECORD_DTYPE).reshape(-1)
        self._ck(self._L.apo_corpus_upload(self._h, _p(recs), recs.shape[0], idx_base))

    def corpus_upload_json(self, text: str | bytes, idx_base: int = 0) -> int:
        """Persisted `senweaver.traceCollector.data` JSON -> Form R -> device corpus; returns T."""
        raw = text.encode() if isinstance(text, str) else text
        n = C.c_uint64(0)
        self._ck(self._L.apo_corpus_upload_json(self._h, raw, len(raw), idx_base, C.byref(n)))
        return n.value

    def corpus_generate(self, seed: int, t0: int, T: int, agent_permille: int = 300):
        self._ck(self._L.apo_corpus_generate(self._h, seed, t0, T, agent_permille))

    def corpus_download(self, first: int, n: int) -> np.ndarray:
        out = np.empty(n, RECORD_DTYPE)
        self._ck(self._L.apo_corpus_download(self._h, _p(out), first, n))
        return out

    # -- evaluations
    def dims_upload(self, dims: np.ndarray):
        dims = np.ascontiguousarray(dims, np.float32)
        Cn, T, nd = dims.shape
        assert nd == NDIM
        self._ck(self._L.apo_dims_upload(self._h, _p(dims), Cn, T))

    def dims_generate(self, seed: int, c0: int, Cn: int, t0: int, T: int, agent_permille: int = 300):
        self._ck(self._L.apo_dims_generate(self._h, seed, c0, Cn, t0, T, agent_permille))

    def dims_download(self, c: int, first: int, n: int) -> np.ndarray:
        out = np.empty((n, NDIM), np.float32)
        self._ck(self._L.apo_dims_download(self._h, _p(out), c, first, n))
        return out

    # Form Q: compact resident layout (12 B per evaluation), lossless for categorical dims
    def dims_compact(self):
        self._ck(self._L.apo_dims_compact(self._h))

    def dims_generate_compact(self, seed: int, c0: int, Cn: int, t0: int, T: int, agent_permille: int = 300):
        self._ck(self._L.apo_dims_generate_compact(self._h, seed, c0, Cn, t0, T, agent_permille))

    def dims_upload_compact(self, dims: np.ndarray):
        dims = np.ascontiguousarray(dims, np.float32)
        Cn, T, nd = dims.shape
        assert nd == NDIM
        self._ck(self._L.apo_dims_upload_compact(self._h, _p(dims), Cn, T))

    def dims_layout(self) -> int:
        """0 nothing loaded, 1 Form D (fp32), 2 Form Q (compact)."""
        return int(self._L.apo_dims_layout(self._h))

    def dims_attach(self, device_ptr: int, Cn: int, T: int, pitch_evals: int):
        self._ck(self._L.apo_dims_attach(self._h, device_ptr, Cn, T, pitch_evals))

    def rollouts_upload(self, recs: np.ndarray):
        recs = np.ascontiguousarray(recs, RECORD_DTYPE)
        Cn, T = recs.shape
        self._ck(self._L.apo_rollouts_upload(self._h, _p(recs), Cn, T))

    def rollouts_generate(self, seed: int, c0: int, Cn: int, t0: int, T: int, agent_permille: int = 300):
        self._ck(self._L.apo_rollouts_generate(self._h, seed, c0, Cn, t0, T, agent_permille))

    def rollouts_download(self, c: int, first: int, n: int) -> np.ndarray:
        out = np.empty(n, RECORD_DTYPE)
        self._ck(self._L.apo_rollouts_download(self._h, _p(out), c, first, n))
        return out

    def rollouts16_upload(self, recs: np.ndarray):
        recs = np.ascontiguousarray(recs, RECORD16_DTYPE)
        Cn, T = recs.shape
        self._ck(self._L.apo_rollouts16_upload(self._h, _p(recs), Cn, T))

    def rollouts16_generate(self, seed: int, c0: int, Cn: int, t0: int, T: int, agent_permille: int = 300):
        self._ck(self._L.apo_rollouts16_generate(self._h, seed, c0, Cn, t0, T, agent_permille))

    def rollouts16_download(self, c: int, first: int, n: int) -> np.ndarray:
        out = np.empty(n, RECORD16_DTYPE)
        self._ck(self._L.apo_rollouts16_download(self._h, _p(out), c, first, n))
        return out

    def score_host_records(self, recs: np.ndarray, K: int, corpus: bool = False, recip: bool = False, variant: int = 0,
                           candidates: bool = False, candidate_corpus: bool = False, extremes: bool = False,
                           groups: bool = False, spread: bool = False, pairs: bool = False, group_pairs: bool = False) -> ScoreResult:
        """recs: C-contiguous [C][T] of RECORD_DTYPE (32 B) or RECORD16_DTYPE (16 B) in host memory."""
        assert recs.flags.c_contiguous and recs.ndim == 2 and recs.dtype.itemsize in (32, 16)
        Cn, T = recs.shape
        o = self._opts(K, SRC_ROLLOUTS, corpus, recip, variant, 0, 0, candidates=candidates, candidate_corpus=candidate_corpus,
                       extremes=extremes, groups=groups, spread=spread, pairs=pairs, group_pairs=group_pairs)
        scores = np.empty(Cn, np.float64)
        counts = np.empty(Cn, np.uint64)
        topk = np.empty(K, np.int32)
        rep = CorpusReport() if corpus else None
        self._ck(self._L.apo_score_host_records(self._h, C.byref(o), _p(recs), recs.dtype.itemsize, Cn, T, _p(scores), _p(counts),
                                                _p(topk), C.byref(rep) if rep is not None else None))
        return ScoreResult(scores, counts, topk, rep, self.last_timing(), self._cands(Cn, candidates),
                           self._ccorp(Cn, candidate_corpus), self._ext(Cn, extremes), self._grp(Cn, groups), self._spr(Cn, spread), self._pairs(Cn, pairs), self._gpairs(Cn, group_pairs))

    # -- scoring
    def _opts(self, K, source, corpus, recip, variant, first, count, timing=False, candidates=False,
              candidate_corpus=False, extremes=False, groups=False, spread=False, pairs=False, group_pairs=False) -> ScoreOpts:
        return ScoreOpts(K, source, (SCORE_CORPUS if corpus else 0) | (SCORE_RECIP if recip else 0) | (SCORE_TIMING if timing else 0)
                         | (SCORE_CANDIDATES if candidates else 0) | (SCORE_CANDIDATE_CORPUS if candidate_corpus else 0)
                         | (SCORE_CANDIDATE_EXTREMES if extremes else 0) | (SCORE_CANDIDATE_GROUPS if groups else 0)
                         | (SCORE_CANDIDATE_SPREAD if spread else 0) | (SCORE_CANDIDATE_PAIRS if pairs else 0)
                         | (SCORE_CANDIDATE_GROUP_PAIRS if group_pairs else 0),
                         variant, first, count)

    def _cands(self, Cn: int, wanted: bool):
        return self.candidate_reports(0, Cn) if wanted else None

    def _ccorp(self, Cn: int, wanted: bool):
        return self.candidate_corpus_reports(0, Cn) if wanted else None

    def _ext(self, Cn: int, wanted: bool):
        return self.candidate_extremes(0, Cn) if wanted else None

    def _grp(self, Cn: int, wanted: bool):
        return self.candidate_groups(0, Cn) if wanted else None

    def _spr(self, Cn: int, wanted: bool):
        return self.candidate_spread(0, Cn) if wanted else None

    def _pairs(self, Cn: int, wanted: bool):
        return self.candidate_pairs(0, Cn) if wanted else None

    def _gpairs(self, Cn: int, wanted: bool):
        return self.candidate_group_pairs(0, Cn) if wanted else None

    def candidate_refs_upload(self, refs):
        """apo_candidate_refs_upload: refs uint32 [C], the reference of every candidate (an index < C, or PAIR_NONE); an empty
        array releases them.  Scoring calls of C candidates with pairs=True then compare every candidate with its reference."""
        refs = np.ascontiguousarray(refs, np.uint32)
        self._ck(self._L.apo_candidate_refs_upload(self._h, _p(refs) if refs.size else None, refs.size))

    def candidate_pairs(self, c0: int, n: int):
        """apo_candidate_pairs: CandidatePair[n] of candidates [c0, c0+n) from the last scoring call, which must have set
        pairs=True (ApoError APO_E_STATE otherwise)."""
        out = (CandidatePair * n)()
        self._ck(self._L.apo_candidate_pairs(self._h, c0, n, out if n else None))
        return out

    def candidate_group_pairs(self, c0: int, n: int, G: int | None = None):
        """apo_candidate_group_pairs: CandidatePair [n][G] of candidates [c0, c0+n) from the last scoring call, which must have
        set group_pairs=True (ApoError APO_E_STATE otherwise): the paired comparison restricted to the record positions of
        each label.  G defaults to the G of the labels held."""
        G = self._groups_G if G is None else G
        out = ((CandidatePair * max(G, 1)) * n)()
        self._ck(self._L.apo_candidate_group_pairs(self._h, c0, n, G, out if n else None))
        return out

    def record_groups_upload(self, labels, G: int = 0):
        """apo_record_groups_upload: labels uint8 [T], the group of every record position (< G <= GROUPS_MAX); an empty
        array releases them.  Scoring calls with groups=True then split every candidate's evaluations by these groups."""
        labels = np.ascontiguousarray(labels, np.uint8).reshape(-1)
        self._ck(self._L.apo_record_groups_upload(self._h, _p(labels) if labels.size else None, labels.size, G))
        self._groups_G = G if labels.size else 0

    def candidate_groups(self, c0: int, n: int, G: int | None = None):
        """apo_candidate_groups: GroupScore [n][G] of candidates [c0, c0+n) from the last scoring call, which must have set
        groups=True (ApoError APO_E_STATE otherwise).  G defaults to the G of the labels held."""
        G = self._groups_G if G is None else G
        out = ((GroupScore * max(G, 1)) * n)()
        self._ck(self._L.apo_candidate_groups(self._h, c0, n, G, out if n else None))
        return out

    def candidate_spread(self, c0: int, n: int):
        """apo_candidate_spread: CandidateSpread[n] of candidates [c0, c0+n) from the last scoring call, which must have set
        spread=True (ApoError APO_E_STATE otherwise)."""
        out = (CandidateSpread * n)()
        self._ck(self._L.apo_candidate_spread(self._h, c0, n, out if n else None))
        return out

    def candidate_extremes(self, c0: int, n: int):
        """apo_candidate_extremes: CandidateExtremes[n] of candidates [c0, c0+n) from the last scoring call, which must have set
        extremes=True (ApoError APO_E_STATE otherwise).  Positions are absolute record positions; each reward is the
        finalReward the call summed."""
        out = (CandidateExtremes * n)()
        self._ck(self._L.apo_candidate_extremes(self._h, c0, n, out if n else None))
        return out

    def candidate_corpus_reports(self, c0: int, n: int):
        """apo_candidate_corpus_reports: CorpusReport[n] of candidates [c0, c0+n) from the last scoring call, which must have
        set candidate_corpus=True (ApoError APO_E_STATE otherwise).  Report c is the corpus report of candidate c's scored
        rollout records (example indices are absolute record positions)."""
        out = (CorpusReport * n)()
        self._ck(self._L.apo_candidate_corpus_reports(self._h, c0, n, out if n else None))
        return out

    def candidate_reports(self, c0: int, n: int):
        """apo_candidate_reports: CandidateReport[n] of candidates [c0, c0+n) from the last scoring call, which must have set
        candidates=True (ApoError APO_E_STATE otherwise)."""
        out = (CandidateReport * n)()
        self._ck(self._L.apo_candidate_reports(self._h, c0, n, out if n else None))
        return out

    def score(self, Cn: int, K: int, source: int = SRC_DIMS, corpus: bool = False, recip: bool = False,
              variant: int = 0, first: int = 0, count: int = 0, timing: bool = False, candidates: bool = False,
              candidate_corpus: bool = False, extremes: bool = False, groups: bool = False, spread: bool = False, pairs: bool = False, group_pairs: bool = False) -> ScoreResult:
        o = self._opts(K, source, corpus, recip, variant, first, count, timing, candidates, candidate_corpus, extremes, groups, spread, pairs, group_pairs)
        scores = np.empty(Cn, np.float64)
        counts = np.empty(Cn, np.uint64)
        topk = np.empty(K, np.int32)
        rep = CorpusReport() if corpus else None
        t = Timing()
        L = self._L
        rc = L.apo_score(self._h, C.byref(o), scores.ctypes.data, counts.ctypes.data, topk.ctypes.data, C.byref(rep) if rep is not None else None)
        if rc != 0:
            self._ck(rc)
        L.apo_last_timing(self._h, C.byref(t))
        return ScoreResult(scores, counts, topk, rep, t, self._cands(Cn, candidates), self._ccorp(Cn, candidate_corpus),
                           self._ext(Cn, extremes), self._grp(Cn, groups), self._spr(Cn, spread), self._pairs(Cn, pairs), self._gpairs(Cn, group_pairs))

    # chunked form: begin / accumulate (per candidate chunk or record window) / finish
    def score_begin(self, C_total: int):
        self._ck(self._L.apo_score_begin(self._h, C_total))

    def score_accumulate(self, cand_offset: int = 0, source: int = SRC_DIMS, recip: bool = False, variant: int = 0,
                         first: int = 0, count: int = 0, candidates: bool = False, candidate_corpus: bool = False,
                         extremes: bool = False, groups: bool = False, spread: bool = False, pairs: bool = False, group_pairs: bool = False):
        o = self._opts(0, source, False, recip, variant, first, count, candidates=candidates, candidate_corpus=candidate_corpus,
                       extremes=extremes, groups=groups, spread=spread, pairs=pairs, group_pairs=group_pairs)
        self._ck(self._L.apo_score_accumulate(self._h, C.byref(o), cand_offset))

    def score_finish(self, C_total: int, K: int, corpus: bool = False, candidates: bool = False,
                     candidate_corpus: bool = False, extremes: bool = False, groups: bool = False, spread: bool = False, pairs: bool = False, group_pairs: bool = False) -> ScoreResult:
        o = self._opts(K, SRC_DIMS, corpus, False, 0, 0, 0, candidates=candidates, candidate_corpus=candidate_corpus, extremes=extremes,
                       groups=groups, spread=spread, pairs=pairs, group_pairs=group_pairs)
        scores = np.empty(C_total, np.float64)
        counts = np.empty(C_total, np.uint64)
        topk = np.empty(K, np.int32)
        rep = CorpusReport() if corpus else None
        self._ck(self._L.apo_score_finish(self._h, C.byref(o), _p(scores), _p(counts), _p(topk),
                                          C.byref(rep) if rep is not None else None))
        return ScoreResult(scores, counts, topk, rep, self.last_timing(), self._cands(C_total, candidates),
                           self._ccorp(C_total, candidate_corpus), self._ext(C_total, extremes), self._grp(C_total, groups),
                           self._spr(C_total, spread), self._pairs(C_total, pairs), self._gpairs(C_total, group_pairs))

    def score_host(self, dims: np.ndarray, K: int, corpus: bool = False, recip: bool = False, variant: int = 0,
                   candidates: bool = False, extremes: bool = False, groups: bool = False, spread: bool = False, pairs: bool = False, group_pairs: bool = False) -> ScoreResult:
        """dims: C-contiguous float32 [C][T][9] in (preferably pinned) host memory."""
        assert dims.dtype == np.float32 and dims.flags.c_contiguous and dims.ndim == 3 and dims.shape[2] == NDIM
        Cn, T, _ = dims.shape
        o = self._opts(K, SRC_DIMS, corpus, recip, variant, 0, 0, candidates=candidates, extremes=extremes, groups=groups, spread=spread, pairs=pairs, group_pairs=group_pairs)
        scores = np.empty(Cn, np.float64)
        counts = np.empty(Cn, np.uint64)
        topk = np.empty(K, np.int32)
        rep = CorpusReport() if corpus else None
        self._ck(self._L.apo_score_host(self._h, C.byref(o), _p(dims), Cn, T, _p(scores), _p(counts), _p(topk),
                                        C.byref(rep) if rep is not None else None))
        return ScoreResult(scores, counts, topk, rep, self.last_timing(), self._cands(Cn, candidates), extremes=self._ext(Cn, extremes),
                           groups=self._grp(Cn, groups), spread=self._spr(Cn, spread), pairs=self._pairs(Cn, pairs), group_pairs=self._gpairs(Cn, group_pairs))

    # -- Form Q in host memory (compact wire format)
    def dims_codebook(self) -> np.ndarray:
        out = np.empty(8 * 256, np.uint32)
        self._ck(self._L.apo_dims_codebook(self._h, _p(out)))
        return out

    def dims_compact_download(self, c: int, first: int, n: int, out=None):
        """(q8 u64[n], d2 f32[n], li u16[n]) of candidate c; pass out=(q8, d2, li) views to fill existing (pinned) buffers."""
        q8, d2, li = out if out is not None else (np.empty(n, np.uint64), np.empty(n, np.float32), np.empty(n, np.uint16))
        self._ck(self._L.apo_dims_compact_download(self._h, _p(q8), _p(d2), _p(li), c, first, n))
        return q8, d2, li

    def score_host_compact(self, q8: np.ndarray, d2: np.ndarray, li: np.ndarray, codebook: np.ndarray, K: int, corpus: bool = False,
                           recip: bool = False, candidates: bool = False, extremes: bool = False,
                          groups: bool = False, spread: bool = False, pairs: bool = False, group_pairs: bool = False) -> ScoreResult:
        """q8 uint64 [C][T], d2 float32 [C][T], li uint16 [C][T] in (preferably pinned) host memory + the uint32[2048] codebook."""
        assert q8.dtype == np.uint64 and d2.dtype == np.float32 and li.dtype == np.uint16 and q8.shape == d2.shape == li.shape and q8.ndim == 2
        assert q8.flags.c_contiguous and d2.flags.c_contiguous and li.flags.c_contiguous
        codebook = np.ascontiguousarray(codebook, np.uint32)
        Cn, T = q8.shape
        o = self._opts(K, SRC_DIMS, corpus, recip, 0, 0, 0, candidates=candidates, extremes=extremes, groups=groups, spread=spread, pairs=pairs, group_pairs=group_pairs)
        scores = np.empty(Cn, np.float64)
        counts = np.empty(Cn, np.uint64)
        topk = np.empty(K, np.int32)
        rep = CorpusReport() if corpus else None
        self._ck(self._L.apo_score_host_compact(self._h, C.byref(o), _p(q8), _p(d2), _p(li), _p(codebook), Cn, T, _p(scores), _p(counts),
                                                _p(topk), C.byref(rep) if rep is not None else None))
        return ScoreResult(scores, counts, topk, rep, self.last_timing(), self._cands(Cn, candidates), extremes=self._ext(Cn, extremes),
                           groups=self._grp(Cn, groups), spread=self._spr(Cn, spread), pairs=self._pairs(Cn, pairs), group_pairs=self._gpairs(Cn, group_pairs))

    def dims_d2book(self) -> np.ndarray:
        out = np.empty(4096, np.uint32)
        self._ck(self._L.apo_dims_d2book(self._h, _p(out)))
        return out

    def dims_packed_download(self, c: int, first: int, n: int, out=None):
        """(pc u32[n], pd u16[n]) of candidate c of the resident compact tensor, in the 6-byte wire format."""
        pc, pd = out if out is not None else (np.empty(n, np.uint32), np.empty(n, np.uint16))
        self._ck(self._L.apo_dims_packed_download(self._h, _p(pc), _p(pd), c, first, n))
        return pc, pd

    def score_host_packed(self, pc: np.ndarray, pd: np.ndarray, codebook: np.ndarray, d2book: np.ndarray, K: int, corpus: bool = False,
                          recip: bool = False, candidates: bool = False, extremes: bool = False,
                          groups: bool = False, spread: bool = False, pairs: bool = False, group_pairs: bool = False) -> ScoreResult:
        """Form P: pc uint32 [C][T] (eight 4-bit codes), pd uint16 [C][T] (tool_success_rate index) + the two codebooks."""
        assert pc.dtype == np.uint32 and pd.dtype == np.uint16 and pc.shape == pd.shape and pc.ndim == 2 and pc.flags.c_contiguous and pd.flags.c_contiguous
        codebook, d2book = np.ascontiguousarray(codebook, np.uint32), np.ascontiguousarray(d2book, np.uint32)
        assert codebook.size == 2048 and d2book.size == 4096
        Cn, T = pc.shape
        o = self._opts(K, SRC_DIMS, corpus, recip, 0, 0, 0, candidates=candidates, extremes=extremes, groups=groups, spread=spread, pairs=pairs, group_pairs=group_pairs)
        scores = np.empty(Cn, np.float64)
        counts = np.empty(Cn, np.uint64)
        topk = np.empty(K, np.int32)
        rep = CorpusReport() if corpus else None
        self._ck(self._L.apo_score_host_packed(self._h, C.byref(o), _p(pc), _p(pd), _p(codebook), _p(d2book), Cn, T, _p(scores), _p(counts),
                                               _p(topk), C.byref(rep) if rep is not None else None))
        return ScoreResult(scores, counts, topk, rep, self.last_timing(), self._cands(Cn, candidates), extremes=self._ext(Cn, extremes),
                           groups=self._grp(Cn, groups), spread=self._spr(Cn, spread), pairs=self._pairs(Cn, pairs), group_pairs=self._gpairs(Cn, group_pairs))

    @staticmethod
    def _tuple_args(tl, th, tbook, codebook, d2book):
        tb_pc, tb_pd = tbook
        assert tl.dtype == np.uint16 and th.dtype == np.uint8 and tl.shape == th.shape and tl.ndim == 2 and tl.flags.c_contiguous and th.flags.c_contiguous
        tb_pc, tb_pd = np.ascontiguousarray(tb_pc, np.uint32), np.ascontiguousarray(tb_pd, np.uint16)
        codebook, d2book = np.ascontiguousarray(codebook, np.uint32), np.ascontiguousarray(d2book, np.uint32)
        assert tb_pc.shape == tb_pd.shape and tb_pc.ndim == 1 and codebook.size == 2048 and d2book.size == 4096
        return tb_pc, tb_pd, codebook, d2book

    def score_host_tuples(self, tl: np.ndarray, th: np.ndarray, tbook, codebook: np.ndarray, d2book: np.ndarray, K: int, corpus: bool = False,
                          recip: bool = False, candidates: bool = False, extremes: bool = False,
                          groups: bool = False, spread: bool = False, pairs: bool = False, group_pairs: bool = False) -> ScoreResult:
        """Form T: tl uint16 [C][T] + th uint8 [C][T] (24-bit dictionary indices), tbook = (pc uint32 [n], pd uint16 [n]) the distinct
        evaluations as Form P pairs, + the two codebooks of Form P."""
        tb_pc, tb_pd, codebook, d2book = self._tuple_args(tl, th, tbook, codebook, d2book)
        Cn, T = tl.shape
        o = self._opts(K, SRC_DIMS, corpus, recip, 0, 0, 0, candidates=candidates, extremes=extremes, groups=groups, spread=spread, pairs=pairs, group_pairs=group_pairs)
        scores = np.empty(Cn, np.float64)
        counts = np.empty(Cn, np.uint64)
        topk = np.empty(K, np.int32)
        rep = CorpusReport() if corpus else None
        self._ck(self._L.apo_score_host_tuples(self._h, C.byref(o), _p(tl), _p(th), _p(tb_pc), _p(tb_pd), tb_pc.size, _p(codebook), _p(d2book), Cn, T,
                                               _p(scores), _p(counts), _p(topk), C.byref(rep) if rep is not None else None))
        return ScoreResult(scores, counts, topk, rep, self.last_timing(), self._cands(Cn, candidates), extremes=self._ext(Cn, extremes),
                           groups=self._grp(Cn, groups), spread=self._spr(Cn, spread), pairs=self._pairs(Cn, pairs), group_pairs=self._gpairs(Cn, group_pairs))

    def tuples_upload(self, tl: np.ndarray, th: np.ndarray, tbook, codebook: np.ndarray, d2book: np.ndarray):
        """Make a Form T tensor resident: score(C, K, source=SRC_TUPLES) then reads 3 B per evaluation."""
        tb_pc, tb_pd, codebook, d2book = self._tuple_args(tl, th, tbook, codebook, d2book)
        Cn, T = tl.shape
        self._ck(self._L.apo_tuples_upload(self._h, _p(tl), _p(th), _p(tb_pc), _p(tb_pd), tb_pc.size, _p(codebook), _p(d2book), Cn, T))

    def dims_tuples(self, cap: int = TUPLES_MAX) -> int:
        """apo_dims_tuples: build resident Form T on the device from the loaded evaluations (their Form W copy or Form Q layout);
        returns the number of dictionary entries.  score(C, K, source=SRC_TUPLES) then reads 3 B per evaluation.  Raises
        ApoError(APO_E_STATE) when the evaluations hold more than `cap` distinct ones (``.n_tuples`` is then a lower bound)."""
        n = C.c_uint32(0)
        rc = self._L.apo_dims_tuples(self._h, cap, C.addressof(n))
        if rc != 0:
            err = ApoError(rc, (self._L.apo_last_error(self._h) or b"").decode())
            err.n_tuples = n.value
            raise err
        return n.value

    def tuples_download(self, c: int, first: int, n: int):
        """(tl uint16[n], th uint8[n]) of candidate c of the resident Form T tensor (built or uploaded)."""
        tl, th = np.empty(n, np.uint16), np.empty(n, np.uint8)
        self._ck(self._L.apo_tuples_download(self._h, _p(tl), _p(th), c, first, n))
        return tl, th

    def tuples_book(self):
        """((tbook_pc, tbook_pd), codebook, d2book) of the resident Form T tensor: the arguments tuples_upload and
        score_host_tuples take besides the planes."""
        n = C.c_uint32(0)
        cb, d2 = np.empty(8 * 256, np.uint32), np.empty(4096, np.uint32)
        rc = self._L.apo_tuples_book(self._h, None, None, 0, _p(cb), _p(d2), C.addressof(n))   # learns n (APO_E_ARG when n > 0)
        if rc != 0 and not (rc == -1 and n.value > 0):
            self._ck(rc)
        pc, pd = np.empty(n.value, np.uint32), np.empty(n.value, np.uint16)
        self._ck(self._L.apo_tuples_book(self._h, _p(pc), _p(pd), n.value, _p(cb), _p(d2), C.addressof(n)))
        return (pc, pd), cb, d2

    def last_timing(self) -> Timing:
        t = Timing()
        self._ck(self._L.apo_last_timing(self._h, C.byref(t)))
        return t

    def debug_partials(self, Cn: int):
        """Exact per-candidate (sum_t rint(finalReward*2^52), count) as Python ints."""
        raw = np.empty((Cn, 4), np.int64)
        self._ck(self._L.apo_debug_partials(self._h, _p(raw), Cn))
        sums = [(int(r[2]) << 64) + (int(r[1]) << 32) + int(r[0]) for r in raw]
        return sums, [int(r[3]) for r in raw]

    def debug_twin_t_list(self):
        """The Form T copy's exception list: (xb [C][blocks per row + 1] uint32 block index, xs [n][2] uint32 {position,
        full index}), or None when no list is held."""
        nw, nx = C.c_uint64(0), C.c_uint64(0)
        self._ck(self._L.apo_debug_twin_t_list(self._h, C.byref(nw), C.byref(nx), None, None))
        if nx.value == 0:
            return None
        xb = np.empty(nw.value, np.uint32)
        xs = np.empty((nx.value, 2), np.uint32)
        self._ck(self._L.apo_debug_twin_t_list(self._h, C.byref(nw), C.byref(nx), _p(xb), _p(xs)))
        return xb, xs

    def debug_twin_h(self):
        """The Form T copy's per-row dictionary counts: (off [C + 1] uint64, pairs [n] uint64 entry | count << 20), or None
        when none are held."""
        rows, nh = C.c_uint32(0), C.c_uint64(0)
        self._ck(self._L.apo_debug_twin_h(self._h, C.byref(rows), C.byref(nh), None, None))
        if nh.value == 0:
            return None
        off = np.empty(rows.value + 1, np.uint64)
        pairs = np.empty(nh.value, np.uint64)
        self._ck(self._L.apo_debug_twin_h(self._h, C.byref(rows), C.byref(nh), _p(off), _p(pairs)))
        return off, pairs

    def debug_corpus_digest(self):
        """The corpus digest: (entries [n][2] uint64 {d2 bits, slots | count << 22}, fixed [45] int64: the tallies, byMode,
        pattern and tool words of the corpus block, then the 18 first-three slots as inverted indices), or None when none
        is held."""
        n = C.c_uint64(0)
        self._ck(self._L.apo_debug_corpus_digest(self._h, C.byref(n), None, None))
        if n.value == 0:
            return None
        ent = np.empty((n.value, 2), np.uint64)
        fixed = np.empty(45, np.int64)
        self._ck(self._L.apo_debug_corpus_digest(self._h, C.byref(n), _p(ent), _p(fixed)))
        return ent, fixed

    # -- multi-GPU
    @staticmethod
    def comm_unique_id() -> bytes:
        L = load_library()
        buf = (C.c_uint8 * UNIQUE_ID_BYTES)()
        rc = L.apo_comm_unique_id(buf)
        if rc != 0:
            raise ApoError(rc, (L.apo_last_error(None) or b"").decode())
        return bytes(buf)

    def comm_init(self, nranks: int, rank: int, uid: bytes):
        assert len(uid) == UNIQUE_ID_BYTES
        buf = (C.c_uint8 * UNIQUE_ID_BYTES).from_buffer_copy(uid)
        self._ck(self._L.apo_comm_init(self._h, nranks, rank, buf))

    def comm_destroy(self):
        self._ck(self._L.apo_comm_destroy(self._h))

    def comm_join_mode(self) -> int:
        """0 single rank, 1 ncclAllReduce join, 2 peer-memory join inside the scoring launch."""
        return int(self._L.apo_comm_join_mode(self._h))


def compact_encode_host(dims: np.ndarray, nthreads: int = 8):
    """Form D float32 [C][T][9] -> (q8, d2, li, codebook): the compact wire format, built on the host (apo_compact_encode_host).
    Raises ApoError(APO_E_STATE) when the data is not categorical."""
    L = load_library()
    dims = np.ascontiguousarray(dims, np.float32)
    Cn, T, nd = dims.shape
    assert nd == NDIM
    q8, d2, li = np.empty((Cn, T), np.uint64), np.empty((Cn, T), np.float32), np.empty((Cn, T), np.uint16)
    book = np.empty(8 * 256, np.uint32)
    rc = L.apo_compact_encode_host(_p(dims), Cn, T, _p(q8), _p(d2), _p(li), _p(book), nthreads)
    if rc != 0:
        raise ApoError(rc, "evaluations are not categorical: a coded dimension has more than 255 distinct values" if rc == -3 else "bad argument")
    return q8, d2, li, book


def packed_encode_host(dims: np.ndarray, nthreads: int = 8, out=None):
    """Form D float32 [C][T][9] -> (pc, pd, codebook, d2book): the 6-byte wire format (apo_packed_encode_host).  out=(pc, pd)
    fills existing (pinned) buffers.  Raises ApoError(APO_E_STATE) when the data does not fit 4-bit / 12-bit codes."""
    L = load_library()
    dims = np.ascontiguousarray(dims, np.float32)
    Cn, T, nd = dims.shape
    assert nd == NDIM
    pc, pd = out if out is not None else (np.empty((Cn, T), np.uint32), np.empty((Cn, T), np.uint16))
    book, d2book = np.empty(8 * 256, np.uint32), np.empty(4096, np.uint32)
    rc = L.apo_packed_encode_host(_p(dims), Cn, T, _p(pc), _p(pd), _p(book), _p(d2book), nthreads)
    if rc != 0:
        raise ApoError(rc, "evaluations do not fit the 4-bit / 12-bit codes of Form P" if rc == -3 else "bad argument")
    return pc, pd, book, d2book


def tuple_encode_host(pc: np.ndarray, pd: np.ndarray, nthreads: int = 8, out=None, cap: int = TUPLES_MAX):
    """Form P planes (pc uint32 [C][T], pd uint16 [C][T]) -> (tl, th, (tbook_pc, tbook_pd)): the 3-byte dictionary form
    (apo_tuple_encode_host).  out=(tl, th) fills existing (pinned) buffers.  Raises ApoError(APO_E_STATE) when the tensor holds
    more than `cap` distinct evaluations."""
    L = load_library()
    assert pc.dtype == np.uint32 and pd.dtype == np.uint16 and pc.shape == pd.shape and pc.ndim == 2 and pc.flags.c_contiguous and pd.flags.c_contiguous
    Cn, T = pc.shape
    tl, th = out if out is not None else (np.empty((Cn, T), np.uint16), np.empty((Cn, T), np.uint8))
    assert tl.dtype == np.uint16 and th.dtype == np.uint8 and tl.shape == pc.shape and th.shape == pc.shape and tl.flags.c_contiguous and th.flags.c_contiguous
    cap = min(int(cap), TUPLES_MAX, max(1, Cn * T))
    tb_pc, tb_pd = np.empty(cap, np.uint32), np.empty(cap, np.uint16)
    n = C.c_uint32(0)
    rc = L.apo_tuple_encode_host(_p(pc), _p(pd), Cn, T, _p(tl), _p(th), _p(tb_pc), _p(tb_pd), cap, C.addressof(n), nthreads)
    if rc != 0:
        raise ApoError(rc, f"{n.value} distinct evaluations exceed the dictionary capacity {cap}" if rc == -3 else "bad argument")
    return tl, th, (tb_pc[:n.value].copy(), tb_pd[:n.value].copy())


def pack16(recs: np.ndarray) -> np.ndarray:
    """Form R -> Form R16 (host helper of the C ABI); raises when a record is not representable."""
    L = load_library()
    recs = np.ascontiguousarray(recs, RECORD_DTYPE)
    out = np.empty(recs.shape, RECORD16_DTYPE)
    bad = C.c_uint64(0)
    rc = L.apo_record_pack16(_p(recs), recs.size, _p(out), C.addressof(bad))
    if rc != 0:
        raise ApoError(rc, f"record {bad.value} is not representable in Form R16")
    return out


def unpack16(recs16: np.ndarray) -> np.ndarray:
    L = load_library()
    recs16 = np.ascontiguousarray(recs16, RECORD16_DTYPE)
    out = np.empty(recs16.shape, RECORD_DTYPE)
    rc = L.apo_record_unpack16(_p(recs16), recs16.size, _p(out))
    if rc != 0:
        raise ApoError(rc, "unpack16 failed")
    return out
