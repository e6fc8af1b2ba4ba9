"""senweaver-ide_b200 — H100-native APO scoring engine (hot path of senweaver/senweaver-ide).

csrc/            sm_90a CUDA kernels + the C ABI (libapo_b200.so, include/apo_b200.h)
engine.py        ctypes binding of the C ABI (plumbing)
sharding.py      record-axis shard arithmetic and the packed partial-vector layout
trace_collector.py / apo_service.py   host-side mirrors of the reference's
                 TraceCollectorService / APOService API that delegate the reductions to the engine

The directory name carries a hyphen (it is the name the build contract fixes), so import it
with importlib:  apo = importlib.import_module("senweaver-ide_b200").
"""
from .engine import (ApoError, CorpusReport, Engine, RECORD_DTYPE, ScoreResult, DIM_NAMES, MODE_NAMES,  # noqa: F401
                     NDIM, NPAT, NMODE, SRC_DIMS, SRC_ROLLOUTS, SRC_TUPLES, TUPLES_MAX, build_library, load_library, LIB_PATH, ABI_SYMBOLS,
                     RECORD16_DTYPE, pack16, unpack16, records_from_json, host_empty, SCORE_TIMING, compact_encode_host, packed_encode_host, tuple_encode_host,
                     TUNE_NO_FUSE, TUNE_FORCE_FUSE, TUNE_NO_STAGING, TUNE_NCCL_JOIN, TUNE_NO_TWIN,
                     TUNE_NO_TWIN_T, TUNE_TWIN_T, TUNE_NO_TWIN_T2, TUNE_NO_TWIN_H, TUNE_NO_CORPUS_DIGEST)
from . import sharding  # noqa: F401
