"""Backend-generic two-fault cases of the ABI's error contract (DESIGN §1, csrc/validate.h): each call gets two bad
arguments at once, and the rule that comes first in the call's audit row wins, with its exact status and text.  The
libraries share one check per call, so the order is one decision; these cases pin it.  Row counts of 2^32 are
passed with one-element columns: a refused call never reads a row."""
import ctypes as C

import numpy as np

from dbsp_b200 import Proj, Schema, Spine, capi, col, key, lval, rval
from dbsp_b200._capi import col_ptrs
from dbsp_b200.zset import _expr, _lanes
from refusal_cases import INVALID, UNSUPPORTED, counters, mutated
from rowfn_cases import _bad

BIG = 1 << 32
ONE = np.array([7], dtype=np.uint64)
W1 = np.array([1], dtype=np.int64)
U_U = Schema("u", "u")
O = C.c_void_p()   # the out-pointer every case passes
RO = C.byref(O)


def expect(be, call, args, status, text):
    """The raw call returns exactly `status` and `text`, touched no out-pointer and launched, copied and waited for
    nothing.  Calls a library does not export are skipped (the plain oracle has no row functions)."""
    if not be.api.exports(call):
        return
    O.value = None
    before = counters(be)
    rc = getattr(be.api, "_" + call)(*args)
    msg = (be.api._last_error() or b"").decode()
    assert (rc, msg) == (status, text), f"{call}: got ({rc}, {msg!r}), expected ({status}, {text!r})"
    assert not O.value, f"{call}: a refused call wrote its out-pointer"
    assert counters(be) == before, f"{call}: a refused call launched, copied or waited"


def bad_proj():
    return mutated(Proj(Schema("u"), [lval(0)]), lambda c: setattr(c, "n_pred", 200))


def fn_of(*out_lanes, fanout=1):
    return Proj(Schema("u" * len(out_lanes)), list(out_lanes), fanout=fanout)


def bad_fn():
    return _bad(fn_of(col(0) % 2), lambda c: setattr(c, "n_insn", 65))


# ---- closures over a raw table: the closure comes before the row count -----------------------------------------------
def case_table_closure_before_rows(be):
    cols = col_ptrs([ONE])
    expect(be, "batch_from_table", (be.ctx, cols, 1, W1.ctypes.data, BIG, 0, bad_proj(), RO),
           INVALID, "batch_from_table: proj.n_pred = 200 exceeds 4")
    expect(be, "batch_from_table_fn", (be.ctx, cols, 1, W1.ctypes.data, BIG, 0, bad_fn(), RO),
           INVALID, "batch_from_table_fn: fn.n_insn = 65 exceeds 64")
    expect(be, "batch_from_table_fanout", (be.ctx, cols, 1, W1.ctypes.data, BIG, 0, bad_fn(), 2, RO),
           INVALID, "batch_from_table_fanout: fn.n_insn = 65 exceeds 64")
    expect(be, "batch_from_table_fanout", (be.ctx, cols, 1, W1.ctypes.data, BIG, 0, fn_of(col(0), fanout=2).c(), 0, RO),
           INVALID, "batch_from_table_fanout: n_out = 0: a fan-out gives 1..64 rows per input row")
    # n_cols before the closure; the columns the closure reads before the row count
    expect(be, "batch_from_table", (be.ctx, cols, 9, W1.ctypes.data, BIG, 0, bad_proj(), RO),
           INVALID, "batch_from_table: n_cols = 9: a table has 1..8 columns")
    expect(be, "batch_from_table", (be.ctx, None, 1, W1.ctypes.data, BIG, 0, Proj(Schema("u"), [lval(0)]).c(), RO),
           INVALID, "batch_from_table: cols is NULL")
    # the row count before the fan-out's rows
    expect(be, "batch_from_table_fanout", (be.ctx, cols, 1, W1.ctypes.data, BIG, 0, fn_of(col(0), fanout=2).c(), 2, RO),
           UNSUPPORTED, "batch_from_table_fanout: n = 4294967296: 2^32-1 or more rows in one batch; split the batch")


# ---- closures over an upload: the upload's context comes before everything it serves ---------------------------------
def case_upload_of_another_context(be):
    other = C.c_void_p()
    assert be.api._ctx_create(0, C.byref(other)) == 0
    up = C.c_void_p()
    try:
        assert be.api._upload_begin(other, col_ptrs([ONE, ONE]), 2, 0b01, W1.ctypes.data, 1, C.byref(up)) == 0
        for call, extra, closure in (("batch_from_upload", (), Proj(Schema("u"), [lval(0)]).c()),
                                     ("batch_from_upload_fn", (), fn_of(col(0) % 2).c()),
                                     ("batch_from_upload_fanout", (2,), fn_of(col(0), fanout=2).c())):
            expect(be, call, (be.ctx, up, closure, *extra, RO), INVALID, f"{call}: upload belongs to another context")
        # with a second fault: a closure that reads a column the upload left out, or a bad n_out
        expect(be, "batch_from_upload", (be.ctx, up, Proj(Schema("u"), [lval(1)]).c(), RO),
               INVALID, "batch_from_upload: upload belongs to another context")
        expect(be, "batch_from_upload_fanout", (be.ctx, up, fn_of(col(0), fanout=2).c(), 0, RO),
               INVALID, "batch_from_upload_fanout: upload belongs to another context")
        # on its own context the upload serves
        expect(be, "batch_from_upload", (other, up, Proj(Schema("u"), [lval(1)]).c(), RO),
               INVALID, "batch_from_upload: proj reads column 1, which col_mask left out of the upload")
    finally:
        be.api._upload_free(up)
        be.api._ctx_destroy(other)


def case_upload_begin(be):
    expect(be, "upload_begin", (be.ctx, None, 9, 0xFF, None, BIG, RO), INVALID, "upload_begin: n_cols = 9: a table has 1..8 columns")
    expect(be, "upload_begin", (be.ctx, col_ptrs([ONE, None]), 2, 0b11, None, BIG, RO), INVALID, "upload_begin: cols[1] is NULL")
    expect(be, "upload_begin", (be.ctx, col_ptrs([ONE, None]), 2, 0b01, None, BIG, RO),
           UNSUPPORTED, "upload_begin: n = 4294967296: 2^32-1 or more rows in one batch; split the batch")


def case_ctx(be):
    expect(be, "ctx_profile", (be.ctx, 3), INVALID, "ctx_profile: enable must be 0, 1 or 2")
    expect(be, "ctx_profile", (be.ctx, -1), INVALID, "ctx_profile: enable must be 0, 1 or 2")
    expect(be, "ctx_profile", (None, 3), INVALID, "ctx_profile: ctx is NULL")
    expect(be, "ctx_create", (-1, None), INVALID, "ctx_create: out is NULL")


# ---- closures over a batch, joins, weigh -------------------------------------------------------------------------------
def case_map_index(be):
    b = be.batch_from_rows(U_U, [(1, 2, 1)])
    expect(be, "map_index", (be.ctx, b.h, bad_proj(), None), INVALID, "map_index: out is NULL")
    expect(be, "map_index", (be.ctx, None, bad_proj(), RO), INVALID, "map_index: batch is NULL")
    expect(be, "map_index_fn", (be.ctx, None, bad_fn(), RO), INVALID, "map_index_fn: batch is NULL")
    expect(be, "map_index_fanout", (be.ctx, b.h, None, 0, RO),
           INVALID, "map_index_fanout: n_out = 0: a fan-out gives 1..64 rows per input row")


def case_join(be):
    a, other = be.batch_from_rows(U_U, [(1, 2, 1)]), be.batch_from_rows(Schema("i", "u"), [(1, 2, 1)])
    tr = Spine(be, Schema("i", "u"))
    differ = "the two inputs differ in key lanes (count or type)"
    p = Proj(Schema("u"), [rval(0)])
    fn = fn_of(rval(0) % 2)
    expect(be, "join_batches", (be.ctx, a.h, other.h, bad_proj(), RO), INVALID, f"join_batches: {differ}")
    expect(be, "join_batches_fn", (be.ctx, a.h, other.h, bad_fn(), RO), INVALID, f"join_batches_fn: {differ}")
    expect(be, "join_delta_trace", (be.ctx, a.h, tr.h, bad_proj(), 0, RO), INVALID, f"join_delta_trace: {differ}")
    expect(be, "join_delta_trace_fn", (be.ctx, a.h, tr.h, bad_fn(), 1, RO), INVALID, f"join_delta_trace_fn: {differ}")
    expect(be, "join_delta_trace", (be.ctx, None, None, p.c(), 1, RO), INVALID, "join_delta_trace: delta is NULL")
    expect(be, "join_batches_fn", (be.ctx, a.h, None, fn.c(), None), INVALID, "join_batches_fn: out is NULL")


def case_weigh(be):
    b, keyless = be.batch_from_rows(U_U, [(1, 2, 1)]), be.batch_empty(Schema("", "u"))
    bad_f = C.byref(_expr(lval(3)).c())
    expect(be, "weigh", (be.ctx, b.h, None, 5, RO), INVALID, "weigh: mode = 5 is not a weigh mode")
    expect(be, "weigh", (be.ctx, keyless.h, bad_f, capi.WEIGH_LINEAR, RO),
           INVALID, "weigh: WEIGH_LINEAR of a batch without key lanes has no output lanes")
    expect(be, "weigh", (be.ctx, None, bad_f, 5, RO), INVALID, "weigh: batch is NULL")
    expect(be, "weigh_fn", (be.ctx, b.h, bad_fn(), 5, RO), INVALID, "weigh_fn: mode = 5 is not a weigh mode")
    expect(be, "weigh_fn", (be.ctx, b.h, fn_of(key(0) % 2, lval(0) % 2).c(), capi.WEIGH_AVG, RO),
           INVALID, "weigh_fn: fn.out_schema must have one lane (the factor)")


# ---- host columns of a schema, two batches of a schema -------------------------------------------------------------------
def case_columns(be):
    sc, bad = U_U.c(), Schema("u", "u").c()
    bad.n_val_lanes = 9
    expect(be, "batch_from_tuples", (be.ctx, C.byref(bad), None, None, BIG, 0, RO),
           INVALID, "batch_from_tuples: schema must have 1..8 lanes, has 1 key + 9 value lanes")
    expect(be, "batch_from_tuples", (be.ctx, C.byref(sc), None, None, BIG, 0, RO), INVALID, "batch_from_tuples: cols is NULL")
    # the weights of sorted rows before their count; a consolidated push counts its rows first
    expect(be, "batch_from_sorted", (be.ctx, C.byref(sc), col_ptrs([ONE, ONE]), None, BIG, 0, RO),
           INVALID, "batch_from_sorted: weights is NULL (consolidated rows carry their weights)")
    q = be.batcher(U_U)
    expect(be, "batcher_push_consolidated", (be.ctx, q.h, col_ptrs([ONE, ONE]), None, BIG, 0),
           UNSUPPORTED, "batcher_push_consolidated: n = 4294967296: 2^32-1 or more rows in one batch; split the batch")
    expect(be, "batcher_push", (be.ctx, None, None, None, BIG, 0), INVALID, "batcher_push: batcher is NULL")
    expect(be, "upsert_commands", (be.ctx, C.byref(sc), None, None, 4, (1 << 63) - 3, 0, RO),
           INVALID, "upsert_commands: seq0 + n = 9223372036854775805 + 4 exceeds 2^63; a command's sequence number has 63 bits")
    expect(be, "upsert_commands", (be.ctx, C.byref(sc), None, None, BIG, 0, 0, RO), INVALID, "upsert_commands: cols is NULL")


def case_pairs(be):
    a, other = be.batch_from_rows(U_U, [(1, 2, 1)]), be.batch_from_rows(Schema("u", "uu"), [(1, 2, 3, 1)])
    tr = Spine(be, U_U)
    for call, args in (("batch_merge", (be.ctx, None, other.h, None)), ("batch_merge_bounded", (be.ctx, None, other.h, None, None)),
                       ("merger_new", (be.ctx, None, other.h, None, None))):
        expect(be, call, args, INVALID, f"{call}: out is NULL")
    expect(be, "batch_merge", (be.ctx, a.h, other.h, RO), INVALID, "batch_merge: a and b differ in schema")
    signed_keyed = be.batch_from_rows(Schema("i", "u"), [(1, 2, 1)])   # other key lanes, and value lanes
    expect(be, "semijoin", (be.ctx, a.h, signed_keyed.h, RO), INVALID, "semijoin: pairs and keys differ in key lanes (count or type)")
    expect(be, "distinct_delta", (be.ctx, other.h, tr.h, None), INVALID, "distinct_delta: out is NULL")
    expect(be, "spine_insert", (be.ctx, None, other.h), INVALID, "spine_insert: spine is NULL")
    expect(be, "window_delta", (be.ctx, tr.h, other.h, 0, None, None, None, None, RO),
           INVALID, "window_delta: trace and delta differ in schema")
    expect(be, "window_delta", (be.ctx, tr.h, a.h, 1, None, None, None, _lanes([7]), RO),
           INVALID, "window_delta: start1 / end1 is NULL")
    expect(be, "aggregate_delta", (be.ctx, a.h, Spine(be, Schema("u", "uu")).h, tr.h, 9, RO),
           INVALID, "aggregate_delta: agg_kind = 9 is not an aggregator")
    expect(be, "aggregate_fold", (be.ctx, a.h, tr.h, None, None, RO), INVALID, "aggregate_fold: out_trace is NULL")
    expect(be, "antijoin_delta", (be.ctx, a.h, Spine(be, Schema("u", "uu")).h, None, None, RO),
           INVALID, "antijoin_delta: key_delta is NULL")
    expect(be, "upsert_delta", (be.ctx, None, None, None), INVALID, "upsert_delta: out is NULL")


# ---- single calls --------------------------------------------------------------------------------------------------------
def case_single(be):
    b = be.batch_from_rows(U_U, [(1, 2, 1)])
    tr = Spine(be, U_U)
    m = be.merger(b, b)
    expect(be, "batch_reindex", (be.ctx, b.h, 9, None), INVALID, "batch_reindex: out is NULL")
    expect(be, "batch_truncate_keys_below", (be.ctx, None, None, RO), INVALID, "batch_truncate_keys_below: batch is NULL")
    expect(be, "spine_truncate_values_below", (be.ctx, None, None), INVALID, "spine_truncate_values_below: spine is NULL")
    expect(be, "batch_last_key", (be.ctx, b.h, None, None), INVALID, "batch_last_key: valid is NULL")
    expect(be, "merger_done", (be.ctx, m.h, None), INVALID, "merger_done: out is NULL")
    expect(be, "shard_partition", (be.ctx, b.h, 0, None), INVALID, "shard_partition: outs is NULL")
    expect(be, "gather", (be.ctx, b.h, 5, None), INVALID, "gather: out is NULL")
    expect(be, "comm_create", (be.ctx, -1, 0, 0, None), INVALID, "comm_create: blob_out is NULL")
    blob = (C.c_uint8 * capi.COMM_BLOB_BYTES)()
    expect(be, "comm_create", (be.ctx, -1, 0, 4096, blob), INVALID, "comm_create: world = 0: 1..32 ranks")
    expect(be, "spine_truncate_keys_below", (be.ctx, tr.h, None), INVALID, "spine_truncate_keys_below: key is NULL")


CASES = {name[5:]: fn for name, fn in globals().items() if name.startswith("case_")}
