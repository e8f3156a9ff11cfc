"""dbsp_b200 — H100-native Z-set delta hot path of DBSP.

Host-side mirror of the reference's Stream/operator API over the C ABI in
include/dbsp_b200.h (CUDA library `libdbsp_b200.so`, sm_90a).  Importable as
`dbsp_b200` through the shim at the repository root.
"""
from . import _capi as capi
from .circuit import Fold, FoldCount, FoldSum, Linear, Max, Min, RootCircuit, Stream, UpsertHandle
from .zset import (After, Backend, Batch, Batcher, Before, Merger, Proj, RelRange, Schema, Spine, acc, col, const, fanout_index, key, lval, rval,
                   val, weight, where_)

__all__ = [
    "capi", "RootCircuit", "Stream", "UpsertHandle", "Max", "Min", "FoldCount", "FoldSum", "Fold", "Backend", "Batch", "Proj",
    "Schema", "Spine", "Batcher", "Merger", "key", "lval", "rval", "val", "col", "const", "where_",
    "fanout_index", "acc", "weight", "Linear", "Before", "After", "RelRange",
]
