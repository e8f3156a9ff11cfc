"""ctypes binding of the C ABI declared in include/dbsp_b200.h.

`CApi(lib, prefix)` binds every entry point of the header.  The product
runtime (`runtime.Runtime`) instantiates it on `libdbsp_b200.so` with the
prefix ``dbsp_``; this module itself contains no compute and no fallback.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

MAX_LANES = 8
MAX_PREDS = 4
MAX_INSNS = 64
MAX_STACK = 16
MAX_FANOUT = 64
MAX_ACC = 15

OK = 0
ERR_NAMES = {1: "DBSP_ERR_INVALID", 2: "DBSP_ERR_CUDA", 3: "DBSP_ERR_NO_DEVICE", 4: "DBSP_ERR_UNSUPPORTED"}

U64, I64 = 0, 1
SRC_KEY, SRC_LVAL, SRC_RVAL, SRC_CONST, SRC_FANOUT, SRC_ACC, SRC_WEIGHT = 0, 1, 2, 3, 4, 5, 6
OP_COPY, OP_NEG, OP_ADD, OP_SUB, OP_MUL, OP_DIV = range(6)
CMP_EQ, CMP_NE, CMP_LT, CMP_LE, CMP_GT, CMP_GE, CMP_IN = range(7)
AGG_MAX, AGG_MIN, AGG_FOLD_COUNT, AGG_FOLD_SUM, AGG_WCOUNT, AGG_WCOUNT2 = range(6)
WEIGH_LINEAR, WEIGH_AVG = 0, 1
ROLLING_LINEAR, ROLLING_MAX, ROLLING_MIN = 0, 1, 2
(FN_PUSH, FN_NEG, FN_ABS, FN_BNOT, FN_LNOT, FN_ADD, FN_SUB, FN_MUL, FN_DIV, FN_REM, FN_DIVU, FN_REMU, FN_MIN, FN_MAX,
 FN_MINU, FN_MAXU, FN_AND, FN_OR, FN_XOR, FN_SHL, FN_SHR, FN_SAR, FN_EQ, FN_NE, FN_LT, FN_LE, FN_GT, FN_GE, FN_LTU,
 FN_LEU, FN_GTU, FN_GEU, FN_IN, FN_SELECT) = range(34)


class CSchema(C.Structure):
    _fields_ = [("n_key_lanes", C.c_uint8), ("n_val_lanes", C.c_uint8), ("lane_types", C.c_uint8 * MAX_LANES)]


class CSrc(C.Structure):
    _fields_ = [("kind", C.c_uint8), ("idx", C.c_uint8), ("pad_", C.c_uint8 * 6), ("cst", C.c_int64)]


class CExpr(C.Structure):
    _fields_ = [("op", C.c_uint8), ("pad_", C.c_uint8 * 7), ("a", CSrc), ("b", CSrc)]


class CPred(C.Structure):
    _fields_ = [("cmp", C.c_uint8), ("is_signed", C.c_uint8), ("pad_", C.c_uint8 * 6), ("a", CSrc), ("b", CSrc)]


class CProj(C.Structure):
    _fields_ = [
        ("out_schema", CSchema),
        ("n_pred", C.c_uint8),
        ("pad_", C.c_uint8 * 5),
        ("out", CExpr * MAX_LANES),
        ("pred", CPred * MAX_PREDS),
    ]


class CInsn(C.Structure):
    _fields_ = [("op", C.c_uint8), ("kind", C.c_uint8), ("idx", C.c_uint8), ("pad_", C.c_uint8 * 5), ("cst", C.c_int64)]


class CRowFn(C.Structure):
    _fields_ = [("out_schema", CSchema), ("n_insn", C.c_uint8), ("pad_", C.c_uint8 * 5), ("code", CInsn * MAX_INSNS)]


class CFold(C.Structure):
    _fields_ = [("n_acc", C.c_uint8), ("n_step", C.c_uint8), ("pad_", C.c_uint8 * 6), ("init", C.c_uint64 * MAX_ACC),
                ("step", CInsn * MAX_INSNS), ("output", CRowFn)]


class CRelRange(C.Structure):
    _fields_ = [("from_after", C.c_uint8), ("to_after", C.c_uint8), ("pad_", C.c_uint8 * 6), ("from_off", C.c_uint64),
                ("to_off", C.c_uint64)]


class DbspError(RuntimeError):
    pass


_P = C.c_void_p
_PP = C.POINTER(C.c_void_p)
_U64P = C.POINTER(C.c_uint64)
_I64P = C.POINTER(C.c_int64)

# name -> argtypes (restype is int32 unless noted)
_SIGS = {
    "ctx_create": [C.c_int32, _PP],
    "ctx_destroy": [_P],
    "ctx_sync": [_P],
    "ctx_stats": [_P, _U64P, _U64P, _U64P, C.c_int32],
    "ctx_profile": [_P, C.c_int32],
    "ctx_profile_read": [_P, C.c_int32, C.c_char_p, _U64P, C.POINTER(C.c_double), _U64P],
    "batch_from_tuples": [_P, C.POINTER(CSchema), _PP, _P, C.c_uint64, C.c_int32, _PP],
    "batch_from_table": [_P, _PP, C.c_uint32, _P, C.c_uint64, C.c_int32, C.POINTER(CProj), _PP],
    "batch_from_sorted": [_P, C.POINTER(CSchema), _PP, _P, C.c_uint64, C.c_int32, _PP],
    "upload_begin": [_P, _PP, C.c_uint32, C.c_uint32, _P, C.c_uint64, _PP],
    "batch_from_upload": [_P, _P, C.POINTER(CProj), _PP],
    "batch_from_table_fn": [_P, _PP, C.c_uint32, _P, C.c_uint64, C.c_int32, C.POINTER(CRowFn), _PP],
    "batch_from_upload_fn": [_P, _P, C.POINTER(CRowFn), _PP],
    "batch_from_table_fanout": [_P, _PP, C.c_uint32, _P, C.c_uint64, C.c_int32, C.POINTER(CRowFn), C.c_uint32, _PP],
    "batch_from_upload_fanout": [_P, _P, C.POINTER(CRowFn), C.c_uint32, _PP],
    "upload_free": [_P],
    "batch_empty": [_P, C.POINTER(CSchema), _PP],
    "batch_merge": [_P, _P, _P, _PP],
    "batcher_new": [_P, C.POINTER(CSchema), _PP],
    "batcher_push": [_P, _P, _PP, _P, C.c_uint64, C.c_int32],
    "batcher_push_consolidated": [_P, _P, _PP, _P, C.c_uint64, C.c_int32],
    "batcher_tuples": [_P, _U64P],
    "batcher_seal": [_P, _P, _PP],
    "batcher_free": [_P],
    "batch_merge_bounded": [_P, _P, _P, _U64P, _PP],
    "merger_new": [_P, _P, _P, _U64P, _PP],
    "merger_work": [_P, _P, _I64P],
    "merger_done": [_P, _P, _PP],
    "merger_free": [_P],
    "batch_truncate_keys_below": [_P, _P, _U64P, _PP],
    "batch_neg": [_P, _P, _PP],
    "batch_reindex": [_P, _P, C.c_uint32, _PP],
    "batch_len": [_P, _U64P],
    "batch_key_count": [_P, _P, _U64P],
    "batch_schema": [_P, C.POINTER(CSchema)],
    "batch_download_csr": [_P, _P, _PP, _P, _PP, _P],
    "batch_download_begin": [_P, _P, _PP, _P, _PP],
    "download_finish": [_P],
    "ctx_sync_stats": [_P, _U64P, C.POINTER(C.c_double), C.c_int32],
    "batch_device_columns": [_P, _PP, _PP],
    "batch_last_key": [_P, _P, _U64P, C.POINTER(C.c_int32)],
    "batch_clone": [_P, _PP],
    "batch_free": [_P],
    "spine_new": [_P, C.POINTER(CSchema), _PP],
    "spine_insert": [_P, _P, _P],
    "spine_consolidate": [_P, _P, _PP],
    "spine_truncate_keys_below": [_P, _P, _U64P],
    "spine_truncate_values_below": [_P, _P, _U64P],
    "spine_exert": [_P, _P, _I64P],
    "spine_len": [_P, _U64P, C.POINTER(C.c_uint32)],
    "spine_free": [_P],
    "spine_save": [_P, _P, C.c_char_p],
    "spine_load": [_P, C.c_char_p, _PP],
    "join_delta_trace": [_P, _P, _P, C.POINTER(CProj), C.c_int32, _PP],
    "join_batches": [_P, _P, _P, C.POINTER(CProj), _PP],
    "join_delta_trace_fn": [_P, _P, _P, C.POINTER(CRowFn), C.c_int32, _PP],
    "join_batches_fn": [_P, _P, _P, C.POINTER(CRowFn), _PP],
    "semijoin": [_P, _P, _P, _PP],
    "aggregate_delta": [_P, _P, _P, _P, C.c_int32, _PP],
    "aggregate_fold": [_P, _P, _P, _P, C.POINTER(CFold), _PP],
    "upsert_commands": [_P, C.POINTER(CSchema), _PP, _P, C.c_uint64, C.c_uint64, C.c_int32, _PP],
    "upsert_delta": [_P, _P, _P, _PP],
    "rolling_aggregate": [_P, _P, _P, _P, C.POINTER(CRelRange), C.c_int32, C.POINTER(CRowFn), _PP],
    "weigh": [_P, _P, C.POINTER(CExpr), C.c_int32, _PP],
    "weigh_fn": [_P, _P, C.POINTER(CRowFn), C.c_int32, _PP],
    "distinct_delta": [_P, _P, _P, _PP],
    "antijoin_delta": [_P, _P, _P, _P, _P, _PP],
    "stream_distinct": [_P, _P, _PP],
    "window_delta": [_P, _P, _P, C.c_int32, _U64P, _U64P, _U64P, _U64P, _PP],
    "map_index": [_P, _P, C.POINTER(CProj), _PP],
    "map_index_fn": [_P, _P, C.POINTER(CRowFn), _PP],
    "map_index_fanout": [_P, _P, C.POINTER(CRowFn), C.c_uint32, _PP],
    "shard_partition": [_P, _P, C.c_uint32, _PP],
    "comm_create": [_P, C.c_int32, C.c_int32, C.c_uint64, _P],
    "comm_connect": [_P, _P],
    "comm_destroy": [_P],
    "comm_info": [_P, C.POINTER(C.c_int32), C.POINTER(C.c_int32), _U64P],
    "shard": [_P, _P, _PP],
    "shard2": [_P, _P, _P, _PP, _PP],
    "gather": [_P, _P, C.c_int32, _PP],
    "allreduce_max_u64": [_P, _U64P],
}
COMM_BLOB_BYTES = 128
# The row-function entry points, fan-outs included.  The CUDA library exports them all; the CPU oracle of the
# dbsp_proj tests (oracle/libdbsp_oracle.so) has none, its row-function build (oracle_fn/libdbsp_oracle_fn.so) has
# them.  A library without them binds every other call, and calling one of them raises DbspError.
ROWFN_CALLS = {"batch_from_table_fn", "batch_from_upload_fn", "join_delta_trace_fn", "join_batches_fn", "weigh_fn",
               "map_index_fn", "batch_from_table_fanout", "batch_from_upload_fanout", "map_index_fanout"}
# Operators added after that oracle: the CUDA library and the row-function oracle export them, the dbsp_proj oracle
# does not.  `CApi.exports` tells a caller which of them a library has.
LATER_CALLS = {"antijoin_delta", "aggregate_fold", "upsert_commands", "upsert_delta", "rolling_aggregate"}


class CApi:
    """Thin, typed view of a shared library exporting the dbsp_b200.h ABI."""

    def __init__(self, lib: C.CDLL, prefix: str):
        self.lib = lib
        self.prefix = prefix
        self.missing = set()
        for name, argtypes in _SIGS.items():
            if name in ROWFN_CALLS | LATER_CALLS and not hasattr(lib, prefix + name):
                self.missing.add(name)
                setattr(self, "_" + name, self._not_exported(prefix + name, name in ROWFN_CALLS))
                continue
            fn = getattr(lib, prefix + name)  # AttributeError if a symbol is missing
            fn.argtypes = argtypes
            fn.restype = C.c_int32
            setattr(self, "_" + name, fn)
        self._last_error = getattr(lib, prefix + "last_error")
        self._last_error.restype = C.c_char_p
        self._last_error.argtypes = []
        self._ctx_stream = getattr(lib, prefix + "ctx_stream")
        self._ctx_stream.restype = C.c_void_p
        self._ctx_stream.argtypes = [_P]
        self._proj_table_mask = getattr(lib, prefix + "proj_table_mask")
        self._proj_table_mask.restype = C.c_uint32
        self._proj_table_mask.argtypes = [C.POINTER(CProj)]
        for mask in ("rowfn_table_mask", "fanout_table_mask"):
            if hasattr(lib, prefix + mask):
                fn = getattr(lib, prefix + mask)
                fn.restype = C.c_uint32
                fn.argtypes = [C.POINTER(CRowFn)]
            else:
                fn = self._not_exported(prefix + mask)
            setattr(self, "_" + mask, fn)

    def exports(self, name: str) -> bool:
        return name not in self.missing

    @staticmethod
    def _not_exported(symbol, rowfn=True):
        def refuse(*_):
            raise DbspError(f"{symbol}: this library has no row functions" if rowfn else f"{symbol}: this library does not export it")
        return refuse

    @staticmethod
    def symbols(prefix: str = "dbsp_"):
        return [prefix + n for n in list(_SIGS) + ["last_error", "ctx_stream", "proj_table_mask", "rowfn_table_mask",
                                                    "fanout_table_mask"]]

    def check(self, rc: int, what: str):
        if rc != OK:
            msg = self._last_error()
            raise DbspError(f"{self.prefix}{what} failed: {ERR_NAMES.get(rc, rc)}: {msg.decode() if msg else ''}")

    def call(self, name: str, *args):
        self.check(getattr(self, "_" + name)(*args), name)


def col_ptrs(cols):
    """Array of void* from a list of numpy arrays / raw integer addresses."""
    arr = (C.c_void_p * max(len(cols), 1))()
    for i, c in enumerate(cols):
        if c is None:
            arr[i] = None
        elif isinstance(c, int):
            arr[i] = c
        else:
            arr[i] = c.ctypes.data
    return arr


def as_u64(a, n=None):
    """Contiguous uint64 view of integer data (i64 lanes are bit-cast)."""
    a = np.asarray(a)
    if a.dtype == np.int64:
        a = a.view(np.uint64)
    elif a.dtype != np.uint64:
        a = a.astype(np.int64).view(np.uint64)
    return np.ascontiguousarray(a)
