"""ctypes mirror of include/rwgpu.h (the C ABI of the H100 HashAgg / HashJoin / shuffle path).

The structs here are a 1:1 transcription of the header; `load_library()` loads the in-tree
`librwgpu.so` and FAILS LOUDLY when it is missing -- there is no CPU fallback in the product.
"""
from __future__ import annotations

import ctypes as C
import os

# ---- status codes
RW_OK = 0
RW_ERR_INVALID = 1
RW_ERR_UNSUPPORTED = 2
RW_ERR_OOM = 3
RW_ERR_NUMERIC_OUT_OF_RANGE = 4
RW_ERR_INCONSISTENT = 5
RW_ERR_CUDA = 6
RW_ERR_NO_DEVICE = 7

# ---- Op (src/common/src/array/stream_chunk.rs:84-91)
OP_INSERT, OP_DELETE, OP_UPDATE_INSERT, OP_UPDATE_DELETE = 1, 2, 3, 4

# ---- types
T_BOOL, T_INT16, T_INT32, T_INT64, T_FLOAT32, T_FLOAT64 = 1, 2, 3, 4, 5, 6
T_DATE, T_TIME, T_TIMESTAMP, T_TIMESTAMPTZ, T_SERIAL, T_DECIMAL = 7, 8, 9, 10, 11, 12
T_VARCHAR, T_BYTEA = 13, 14  # varlen payload: offsets[n + 1] + bytes
VARLEN_TYPES = (T_VARCHAR, T_BYTEA)

TYPE_WIDTH = {T_BOOL: 1, T_INT16: 2, T_INT32: 4, T_INT64: 8, T_FLOAT32: 4, T_FLOAT64: 8, T_DATE: 4,
              T_TIME: 8, T_TIMESTAMP: 8, T_TIMESTAMPTZ: 8, T_SERIAL: 8, T_DECIMAL: 16}

# ---- agg kinds / join types / sides / cmp
AGG_COUNT, AGG_SUM, AGG_MIN, AGG_MAX, AGG_SUM0 = 1, 2, 3, 4, 5
(JOIN_INNER, JOIN_LEFT_OUTER, JOIN_RIGHT_OUTER, JOIN_FULL_OUTER, JOIN_LEFT_SEMI, JOIN_LEFT_ANTI,
 JOIN_RIGHT_SEMI, JOIN_RIGHT_ANTI) = range(8)
SIDE_LEFT, SIDE_RIGHT = 0, 1
CMP_NONE, CMP_LT, CMP_LE, CMP_GT, CMP_GE, CMP_EQ, CMP_NE = range(7)


class RwColumn(C.Structure):
    _fields_ = [("type", C.c_int32), ("reserved", C.c_int32), ("data", C.c_void_p),
                ("validity", C.c_void_p), ("offsets", C.c_void_p)]


class RwChunk(C.Structure):
    _fields_ = [("n_rows", C.c_int64), ("n_cols", C.c_int32), ("reserved", C.c_int32),
                ("ops", C.c_void_p), ("visibility", C.c_void_p), ("columns", C.POINTER(RwColumn))]


class RwAggCall(C.Structure):
    _fields_ = [("kind", C.c_int32), ("arg_col", C.c_int32), ("ret_type", C.c_int32),
                ("reserved", C.c_int32)]


class RwAggDesc(C.Structure):
    _fields_ = [("n_input_cols", C.c_int32), ("input_types", C.POINTER(C.c_int32)),
                ("n_group_keys", C.c_int32), ("group_key_indices", C.POINTER(C.c_int32)),
                ("n_calls", C.c_int32), ("calls", C.POINTER(RwAggCall)),
                ("row_count_index", C.c_int32), ("is_append_only", C.c_int32),
                ("chunk_size", C.c_int32), ("strict_consistency", C.c_int32),
                ("group_capacity_hint", C.c_uint64)]


class RwJoinCond(C.Structure):
    _fields_ = [("cmp", C.c_int32), ("lhs", C.c_int32), ("rhs", C.c_int32), ("reserved", C.c_int32)]


class RwFilterTerm(C.Structure):
    _fields_ = [("cmp", C.c_int32), ("lhs_col", C.c_int32), ("rhs_col", C.c_int32), ("reserved", C.c_int32),
                ("rhs_const", C.c_int64)]


class RwExprOp(C.Structure):
    _fields_ = [("op", C.c_int32), ("arg", C.c_int32), ("value", C.c_int64)]


class RwProjectExpr(C.Structure):
    _fields_ = [("ops", C.POINTER(RwExprOp)), ("n_ops", C.c_int32), ("ret_type", C.c_int32)]


EX_COL, EX_CONST, EX_ADD, EX_SUB, EX_MUL, EX_DIV, EX_MOD, EX_TUMBLE_START, EX_TUMBLE_END, EX_NEG = range(1, 11)


class RwJoinSideDesc(C.Structure):
    _fields_ = [("n_cols", C.c_int32), ("types", C.POINTER(C.c_int32)),
                ("key_indices", C.POINTER(C.c_int32)),
                ("n_pk", C.c_int32), ("pk_indices", C.POINTER(C.c_int32)),
                ("n_stream_key", C.c_int32), ("stream_key", C.POINTER(C.c_int32)),
                ("row_capacity_hint", C.c_uint64), ("stored_rows_hint", C.c_uint64)]


class RwJoinDesc(C.Structure):
    _fields_ = [("join_type", C.c_int32), ("n_keys", C.c_int32),
                ("left", RwJoinSideDesc), ("right", RwJoinSideDesc),
                ("null_safe", C.POINTER(C.c_uint8)),
                ("n_output", C.c_int32), ("output_indices", C.POINTER(C.c_int32)),
                ("cond", RwJoinCond),
                ("is_append_only", C.c_int32), ("chunk_size", C.c_int32),
                ("strict_consistency", C.c_int32), ("reserved", C.c_int32)]


class RwError(RuntimeError):
    """Non-zero status from the C ABI; `.code` is the RW_ERR_* value
    (maps to StreamExecutorError in the Rust shim, SURVEY §8b)."""

    def __init__(self, code: int, msg: str):
        super().__init__(f"rwgpu status {code}: {msg}")
        self.code = code


_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "librwgpu.so")
_lib = None


def load_library() -> C.CDLL:
    """Load the in-tree CUDA library.  Raises (never falls back) if it is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc -gencode arch=compute_90a,code=sm_90a). There is no CPU fallback.")
        _lib = C.CDLL(LIB_PATH)
    return _lib


# every symbol include/rwgpu.h declares (checked by tests/test_abi.py)
ABI_SYMBOLS = [
    "rwgpu_type_width", "rwgpu_out_num_chunks", "rwgpu_out_num_rows", "rwgpu_out_chunk",
    "rwgpu_out_release", "rwgpu_agg_create", "rwgpu_agg_destroy", "rwgpu_agg_push",
    "rwgpu_agg_push_device", "rwgpu_agg_push_device_counted", "rwgpu_agg_flush", "rwgpu_agg_flush_device", "rwgpu_agg_flush_device_async", "rwgpu_agg_flush_collect", "rwgpu_agg_stats", "rwgpu_agg_profile", "rwgpu_agg_snapshot", "rwgpu_agg_restore",
    "rwgpu_agg_update_watermark", "rwgpu_agg_value_log_stats",
    "rwgpu_join_create", "rwgpu_join_destroy", "rwgpu_join_push", "rwgpu_join_push_device", "rwgpu_join_push_device_counted", "rwgpu_join_push_device_async", "rwgpu_join_collect", "rwgpu_join_push_async", "rwgpu_join_collect_out",
    "rwgpu_join_barrier", "rwgpu_join_stats", "rwgpu_join_profile", "rwgpu_join_debug_set_seq", "rwgpu_join_snapshot", "rwgpu_join_restore", "rwgpu_join_update_watermark", "rwgpu_join_compactions", "rwgpu_vnode_compute", "rwgpu_dispatch_rewrite_ops",
    "rwgpu_shuffle_partition_device", "rwgpu_shuffle_p2p_region_bytes",
    "rwgpu_shuffle_partition_p2p_device", "rwgpu_shuffle_unpack_device", "rwgpu_shuffle_exchange_p2p_device", "rwgpu_shuffle_flat_layout", "rwgpu_shuffle_exchange_flat_device", "rwgpu_filter", "rwgpu_filter_device", "rwgpu_project", "rwgpu_project_device", "rwgpu_last_error", "rwgpu_device_check", "rwgpu_version",
]
