/*
 * dbsp_b200.h — C ABI of the H100-native Z-set delta hot path.
 *
 * This is the drop-in boundary for the path BASELINE.json's north_star names:
 * the reference's `Batch` / `Batcher` / `Builder` / `Merger` / `Trace` trait
 * family (crates/dbsp/src/trace/mod.rs:86-396) and the `eval` bodies of the
 * relational operators that consume it.  A Rust `dbsp-b200-sys` crate binds
 * exactly these symbols (see INTEGRATION.md); all arguments are plain
 * pointers, sizes and POD structs — no torch / C++ types cross the boundary.
 *
 * Conventions (mirroring SURVEY.md §8b):
 *   - every call returns int32 status, 0 = DBSP_OK; no exception crosses;
 *   - a `dbsp_ctx` is bound to one GPU + one CUDA stream and must be used
 *     from one host thread at a time (the reference confines a circuit
 *     replica to its worker thread, circuit_builder.rs:1439-1450);
 *   - batches are immutable, reference counted values (the reference's
 *     batches are immutable values too, zset_batch.rs:27);
 *   - every *_free (and dbsp_download_finish) is a no-op on NULL.
 *
 * Error contract.  Every argument is checked on the host before the call
 * allocates, copies or launches anything.  A refused call returns
 * DBSP_ERR_INVALID (DBSP_ERR_UNSUPPORTED for 2^32-1 or more rows in one
 * batch), leaves a dbsp_last_error text naming the call and the argument,
 * writes no out-pointer and leaves the context and its handles usable.
 * Refused everywhere: a NULL context, a NULL handle, a NULL in- or out-pointer
 * that a comment below does not call optional; a schema without 1..8 lanes
 * or with a lane type other than DBSP_U64 / DBSP_I64; a row expression whose
 * kind / op / cmp is outside its enum, whose n_pred exceeds DBSP_MAX_PREDS or
 * whose idx is not below the lane count of the source it names; a row
 * function with more than DBSP_MAX_INSNS instructions, an op or a PUSH kind
 * outside its enum, a PUSH idx not below the lane count of its source, a stack
 * that underflows or grows past DBSP_MAX_STACK, or a final depth other than
 * the output lanes + 1 (checked in O(n_insn)); two operands
 * whose schemas do not fit each other (noted per call).  DESIGN.md §1 lists
 * the checks of every entry point.
 *
 * Data model.  A row is `n_key_lanes + n_val_lanes` 64-bit lanes plus one
 * int64 weight.  Lanes are u64 or i64 and compare lexicographically, which
 * is Rust's derived `Ord` on tuples of integers.  `n_val_lanes == 0` is an
 * `OrdZSet<K,R>` (zset_batch.rs:28-31); otherwise an
 * `OrdIndexedZSet<K,V,R>` (indexed_zset_batch.rs:27-41).  On the device a
 * batch is column-major: one contiguous u64 array per lane plus the weight
 * array, rows sorted by (key lanes, val lanes), consolidated (no duplicate
 * rows, no zero weights).  `dbsp_batch_download_csr` returns the
 * reference's canonical `keys / offs / vals / diffs` vectors.
 */
#ifndef DBSP_B200_H
#define DBSP_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DBSP_MAX_LANES 8
#define DBSP_MAX_PREDS 4

enum dbsp_status {
  DBSP_OK = 0,
  DBSP_ERR_INVALID = 1,   /* bad argument / schema mismatch                */
  DBSP_ERR_CUDA = 2,      /* CUDA runtime error (see dbsp_last_error)      */
  DBSP_ERR_NO_DEVICE = 3, /* no usable CUDA device: there is NO CPU fallback */
  DBSP_ERR_UNSUPPORTED = 4
};

enum dbsp_lane_type { DBSP_U64 = 0, DBSP_I64 = 1 };

/* Row schema.  Replaces the `K: DBData, V: DBData` type parameters of
 * `Batch` (trace/mod.rs:49-76, 237-300) for the supported key/value set:
 * tuples of <= 8 integer lanes in total. */
typedef struct dbsp_schema {
  uint8_t n_key_lanes;
  uint8_t n_val_lanes;
  uint8_t lane_types[DBSP_MAX_LANES]; /* key lanes first, then val lanes */
} dbsp_schema;

/* ---- declarative row expressions (replace the Rust closures passed to
 * join / flat_map_index / map_index, join.rs:187, filter_map.rs:143-152) -- */
enum dbsp_src_kind {
  DBSP_SRC_KEY = 0,   /* lane `idx` of the (join) key                       */
  DBSP_SRC_LVAL = 1,  /* lane `idx` of the left value (v1 of join_func);
                         for map_index / raw tables: value lane / column    */
  DBSP_SRC_RVAL = 2,  /* lane `idx` of the right value (v2 of join_func);
                         in a call with one input: the same lanes as LVAL  */
  DBSP_SRC_CONST = 3, /* the constant `cst`                                 */
  DBSP_SRC_FANOUT = 4,/* row functions of the `_fanout` calls only: j, the
                         index (0 .. n_out-1) of the output being generated;
                         idx and cst are ignored.  Every other call refuses
                         it as outside the enum.                            */
  DBSP_SRC_ACC = 5,   /* the programs of a dbsp_fold only: accumulator word
                         `idx` (< n_acc)                                     */
  DBSP_SRC_WEIGHT = 6 /* a dbsp_fold's step only: the value's weight (summed
                         over the trace's batches) as i64 bits; idx and cst
                         are ignored                                         */
};
enum dbsp_expr_op {
  DBSP_OP_COPY = 0, DBSP_OP_NEG = 1, DBSP_OP_ADD = 2, DBSP_OP_SUB = 3,
  DBSP_OP_MUL = 4,
  DBSP_OP_DIV = 5 /* signed, truncating (Rust isize `/`), wrapping: x / 0 = 0
                     and MIN / -1 = MIN (i64::wrapping_div); NEG/ADD/SUB/MUL
                     wrap mod 2^64 */
};
enum dbsp_cmp_op {
  DBSP_CMP_EQ = 0, DBSP_CMP_NE = 1, DBSP_CMP_LT = 2, DBSP_CMP_LE = 3,
  DBSP_CMP_GT = 4, DBSP_CMP_GE = 5,
  DBSP_CMP_IN = 6 /* a < 64 && bit a of b is set: membership in a small code
                     set, e.g. STATES_OF_INTEREST.contains (nexmark q3.rs:44) */
};
typedef struct dbsp_src {
  uint8_t kind;
  uint8_t idx;
  uint8_t pad_[6];
  int64_t cst;
} dbsp_src;
typedef struct dbsp_expr {
  uint8_t op;
  uint8_t pad_[7];
  dbsp_src a, b;
} dbsp_expr;
typedef struct dbsp_pred {
  uint8_t cmp;
  uint8_t is_signed;
  uint8_t pad_[6];
  dbsp_src a, b;
} dbsp_pred;
/* Projection + filter: output row = (out[0..n_out_key+n_out_val)), kept iff
 * every predicate holds. */
typedef struct dbsp_proj {
  dbsp_schema out_schema;
  uint8_t n_pred;
  uint8_t pad_[5];
  dbsp_expr out[DBSP_MAX_LANES];
  dbsp_pred pred[DBSP_MAX_PREDS];
} dbsp_proj;

/* Row functions: closures that are expression trees (nested arithmetic, remainders, bitwise ops, conditionals,
 * predicates combined with AND / OR / NOT), the second closure form, accepted by the `_fn` twins of the calls that
 * take a dbsp_proj.  A program is postfix over a stack of u64 values, at most DBSP_MAX_STACK deep: PUSH pushes the
 * source `kind` / `idx` / `cst` (the meaning of dbsp_src); every other instruction pops its operands (the last
 * pushed is the right-hand one) and pushes one result, and ignores kind, idx and cst.  When the program ends the
 * stack holds exactly L + 1 values, L = the lane count of out_schema: the output lanes in order, then the keep
 * flag (non-zero = keep the row).  Every operation is total (wrapping, no trap).  DESIGN.md §2 defines them. */
#define DBSP_MAX_INSNS 64
#define DBSP_MAX_STACK 16
enum dbsp_fn_op {
  DBSP_FN_PUSH = 0,
  /* unary */
  DBSP_FN_NEG = 1, DBSP_FN_ABS = 2 /* wrapping_abs: ABS(MIN) = MIN */, DBSP_FN_BNOT = 3, DBSP_FN_LNOT = 4 /* x == 0 */,
  /* binary */
  DBSP_FN_ADD = 5, DBSP_FN_SUB = 6, DBSP_FN_MUL = 7,
  DBSP_FN_DIV = 8, DBSP_FN_REM = 9,    /* signed, wrapping: x / 0 = x % 0 = 0, MIN / -1 = MIN, MIN % -1 = 0 */
  DBSP_FN_DIVU = 10, DBSP_FN_REMU = 11, /* u64: x / 0 = x % 0 = 0 */
  DBSP_FN_MIN = 12, DBSP_FN_MAX = 13, DBSP_FN_MINU = 14, DBSP_FN_MAXU = 15,
  DBSP_FN_AND = 16, DBSP_FN_OR = 17, DBSP_FN_XOR = 18,
  DBSP_FN_SHL = 19, DBSP_FN_SHR = 20, DBSP_FN_SAR = 21, /* count mod 64 (wrapping_shl / _shr) */
  /* comparisons: 0 or 1 */
  DBSP_FN_EQ = 22, DBSP_FN_NE = 23,
  DBSP_FN_LT = 24, DBSP_FN_LE = 25, DBSP_FN_GT = 26, DBSP_FN_GE = 27,     /* signed   */
  DBSP_FN_LTU = 28, DBSP_FN_LEU = 29, DBSP_FN_GTU = 30, DBSP_FN_GEU = 31, /* unsigned */
  DBSP_FN_IN = 32,    /* a < 64 && bit a of b is set (DBSP_CMP_IN) */
  /* ternary */
  DBSP_FN_SELECT = 33 /* c, a, b -> c != 0 ? a : b */
};
typedef struct dbsp_insn {
  uint8_t op;   /* dbsp_fn_op */
  uint8_t kind; /* PUSH: dbsp_src_kind */
  uint8_t idx;  /* PUSH: lane / column */
  uint8_t pad_[5];
  int64_t cst;  /* PUSH of DBSP_SRC_CONST */
} dbsp_insn;
typedef struct dbsp_rowfn {
  dbsp_schema out_schema;
  uint8_t n_insn;
  uint8_t pad_[5];
  dbsp_insn code[DBSP_MAX_INSNS];
} dbsp_rowfn;

/* A Fold aggregator (operator/aggregate/fold.rs: Fold::new / with_output) as
 * two row-function programs over an accumulator of n_acc untyped u64 words:
 *   init    the accumulator's first value (Fold::init; words >= n_acc unused);
 *   step    Fold::step(&mut acc, &value, weight), n_step instructions over
 *           KEY / LVAL (RVAL = LVAL) of the value's row, ACC, WEIGHT and
 *           CONST; it ends with the n_acc new words, then a keep flag: 0 leaves
 *           acc unchanged, non-zero replaces it with the new words;
 *   output  Fold's output function, a dbsp_rowfn over KEY, ACC and CONST whose
 *           out_schema has only value lanes (the aggregate's values); a keep
 *           flag of 0 gives the key no output row.
 * The accumulator plus the keep flag fit the DBSP_MAX_STACK-deep stack. */
#define DBSP_MAX_ACC 15
typedef struct dbsp_fold {
  uint8_t n_acc;                    /* 1..DBSP_MAX_ACC */
  uint8_t n_step;                   /* instructions in step[], <= DBSP_MAX_INSNS */
  uint8_t pad_[6];
  uint64_t init[DBSP_MAX_ACC];
  dbsp_insn step[DBSP_MAX_INSNS];
  dbsp_rowfn output;
} dbsp_fold;

/* Aggregators (operator/aggregate/{max,min,fold}.rs, mod.rs:129-156). */
enum dbsp_agg_kind {
  DBSP_AGG_MAX = 0,        /* Max over the value tuple  (max.rs:36-55)       */
  DBSP_AGG_MIN = 1,        /* Min                       (min.rs:38-57)       */
  DBSP_AGG_FOLD_COUNT = 2, /* Fold: # values with non-zero weight            */
  DBSP_AGG_FOLD_SUM = 3,   /* Fold: sum of value lane 0 over such values     */
  DBSP_AGG_WCOUNT = 4,     /* WeightedCount over OrdZSet<K> (mod.rs:129-156) */
  DBSP_AGG_WCOUNT2 = 5     /* WeightedCount over the (sum,count) pair weight
                              of `average` (average.rs:26-29): delta is
                              OrdZSet<(K.., which)>, which in {0,1}          */
};
enum dbsp_weigh_mode {
  DBSP_WEIGH_LINEAR = 0, /* weigh(f): weight_k = sum f(k,v)*w (mod.rs:297-323) */
  DBSP_WEIGH_AVG = 1     /* f = Avg(value,1): rows (k,0)->sum v*w, (k,1)->sum w */
};

typedef struct dbsp_ctx dbsp_ctx;
typedef struct dbsp_batch dbsp_batch;
typedef struct dbsp_spine dbsp_spine;

/* ---- context -------------------------------------------------------- */
/* One context per GPU / circuit replica (runtime.rs:137-180: one worker =
 * one replica).  Fails with DBSP_ERR_NO_DEVICE when no CUDA device is
 * usable — there is no CPU path behind this ABI. */
int32_t dbsp_ctx_create(int32_t device, dbsp_ctx** out);
int32_t dbsp_ctx_destroy(dbsp_ctx* ctx);
int32_t dbsp_ctx_sync(dbsp_ctx* ctx);
const char* dbsp_last_error(void);
/* Counters: kernels launched by this library and bytes it copied H2D/D2H
 * since the last reset (bench.py's gpu_launches / e2e byte counts). */
int32_t dbsp_ctx_stats(dbsp_ctx* ctx, uint64_t* kernel_launches,
                       uint64_t* h2d_bytes, uint64_t* d2h_bytes, int32_t reset);
/* Optional per-kernel timing (CUDA events on the context's stream around the
 * library's own kernels).  enable == 1 starts a fresh collection, enable == 2
 * pauses it (what was collected stays readable, nothing more is recorded —
 * a sampling window inside a longer timed region), enable == 0 ends it.  _read
 * returns, for kernel class `kernel_id` (0,1,2,... until DBSP_ERR_INVALID),
 * its name, launch count, summed device time and algorithmic bytes (the
 * per-kernel byte formulas of DESIGN.md). */
int32_t dbsp_ctx_profile(dbsp_ctx* ctx, int32_t enable);
int32_t dbsp_ctx_profile_read(dbsp_ctx* ctx, int32_t kernel_id, char* name32,
                              uint64_t* launches, double* ms,
                              uint64_t* alg_bytes);
/* CUDA stream the context launches on (cudaStream_t as void*), so a host
 * can order its own work / CUDA events on it. */
void* dbsp_ctx_stream(dbsp_ctx* ctx);

/* ---- batches -------------------------------------------------------- */
/* Batch::from_tuples (trace/mod.rs:259-263) = MergeBatcher + consolidate
 * (merge_batcher/mod.rs:65-80,155-197; consolidation/mod.rs:32-52) + Builder
 * (ordered/mod.rs:874-888): sort, sum equal rows, drop zero weights.
 * `cols[l]` points to n u64 per lane (key lanes then val lanes); `weights`
 * may be NULL (all +1).  `on_device` != 0: the pointers are device memory. */
int32_t dbsp_batch_from_tuples(dbsp_ctx* ctx, const dbsp_schema* schema,
                               const uint64_t* const* cols,
                               const int64_t* weights, uint64_t n,
                               int32_t on_device, dbsp_batch** out);
/* flat_map_index over a raw (unsorted, column-major) event table followed by
 * from_tuples (filter_map.rs:700-724): every source kind names a column,
 * idx < n_cols (1..8).  Only the columns `proj` reads need be non-NULL. */
int32_t dbsp_batch_from_table(dbsp_ctx* ctx, const uint64_t* const* cols,
                              uint32_t n_cols, const int64_t* weights,
                              uint64_t n, int32_t on_device,
                              const dbsp_proj* proj, dbsp_batch** out);
/* Pipelined ingest of a raw event table: start copying the host columns of a
 * *future* step to the device on the context's copy stream (pinned host
 * memory makes it overlap with the kernels of the current step); the handle
 * is then consumed by dbsp_batch_from_upload.  `col_mask` bit l = column l is
 * needed (the others are not copied).  The host buffers must stay valid until
 * the upload is consumed or freed.  dbsp_batch_from_upload refuses a `proj`
 * that reads a column outside `col_mask`.  This is the double-buffered input queue of
 * the reference's source operators (crates/nexmark/src/lib.rs:105-231 feeds
 * batches ahead of the circuit) moved to the PCIe boundary. */
typedef struct dbsp_upload dbsp_upload;
int32_t dbsp_upload_begin(dbsp_ctx* ctx, const uint64_t* const* cols,
                          uint32_t n_cols, uint32_t col_mask,
                          const int64_t* weights, uint64_t n,
                          dbsp_upload** out);
int32_t dbsp_batch_from_upload(dbsp_ctx* ctx, dbsp_upload* up,
                               const dbsp_proj* proj, dbsp_batch** out);
int32_t dbsp_upload_free(dbsp_upload* up);
/* Columns of the table a projection reads (bit l = a source with idx l);
 * 0 for a NULL or malformed projection.  Needs no context. */
uint32_t dbsp_proj_table_mask(const dbsp_proj* proj);
/* The same three calls with a row function (dbsp_rowfn) as the closure. */
int32_t dbsp_batch_from_table_fn(dbsp_ctx* ctx, const uint64_t* const* cols,
                                 uint32_t n_cols, const int64_t* weights,
                                 uint64_t n, int32_t on_device,
                                 const dbsp_rowfn* fn, dbsp_batch** out);
int32_t dbsp_batch_from_upload_fn(dbsp_ctx* ctx, dbsp_upload* up,
                                  const dbsp_rowfn* fn, dbsp_batch** out);
uint32_t dbsp_rowfn_table_mask(const dbsp_rowfn* fn);
/* Fan-out (flat_map returning an iterator, filter_map.rs:124-160): the row
 * function runs n_out times per input row, with j = 0 .. n_out-1 pushed by
 * DBSP_SRC_FANOUT; input row i yields output j iff the keep flag of run j is
 * non-zero.  Every output row carries the weight of its input row, and the
 * result is consolidated like every other output.  1 <= n_out <=
 * DBSP_MAX_FANOUT (else INVALID); rows * n_out of 2^32-1 or more is
 * UNSUPPORTED, checked from the sizes before anything runs.  The table, upload
 * and batch forms take what batch_from_table_fn / batch_from_upload_fn /
 * map_index_fn take, and fanout_table_mask is rowfn_table_mask with FANOUT
 * pushes allowed (they read no column). */
#define DBSP_MAX_FANOUT 64
int32_t dbsp_batch_from_table_fanout(dbsp_ctx* ctx, const uint64_t* const* cols,
                                     uint32_t n_cols, const int64_t* weights,
                                     uint64_t n, int32_t on_device,
                                     const dbsp_rowfn* fn, uint32_t n_out,
                                     dbsp_batch** out);
int32_t dbsp_batch_from_upload_fanout(dbsp_ctx* ctx, dbsp_upload* up,
                                      const dbsp_rowfn* fn, uint32_t n_out,
                                      dbsp_batch** out);
uint32_t dbsp_fanout_table_mask(const dbsp_rowfn* fn);
int32_t dbsp_batch_empty(dbsp_ctx* ctx, const dbsp_schema* schema,
                         dbsp_batch** out);
/* Batch::merge / Merger::work run to completion (trace/mod.rs:371-396;
 * column_layer/builders.rs:98-169; ordered/mod.rs:344-396,806-834). */
int32_t dbsp_batch_merge(dbsp_ctx* ctx, const dbsp_batch* a,
                         const dbsp_batch* b, dbsp_batch** out);
/* Batcher (trace/mod.rs:316-335) = MergeBatcher (trace/ord/merge_batcher/mod.rs:22-81,
 * 155-260): push_batch consolidates the pushed tuples and queues them, merging
 * the two newest queue entries while the newer is at least half the older;
 * push_consolidated skips the consolidation (rows already sorted, unique, non-zero);
 * seal merges what is left into one batch and frees the batcher. */
typedef struct dbsp_batcher dbsp_batcher;
int32_t dbsp_batcher_new(dbsp_ctx* ctx, const dbsp_schema* schema,
                         dbsp_batcher** out);
int32_t dbsp_batcher_push(dbsp_ctx* ctx, dbsp_batcher* b,
                          const uint64_t* const* cols, const int64_t* weights,
                          uint64_t n, int32_t on_device);
int32_t dbsp_batcher_push_consolidated(dbsp_ctx* ctx, dbsp_batcher* b,
                                       const uint64_t* const* cols,
                                       const int64_t* weights, uint64_t n,
                                       int32_t on_device);
int32_t dbsp_batcher_tuples(const dbsp_batcher* b, uint64_t* n_tuples);
int32_t dbsp_batcher_seal(dbsp_ctx* ctx, dbsp_batcher* b, dbsp_batch** out);
int32_t dbsp_batcher_free(dbsp_batcher* b);
/* Merger::work with a lower value bound, run to completion
 * (trace/ord/indexed_zset_batch.rs:359-382 -> ordered/mod.rs:587-746
 * push_merge_truncate_values_fueled): values below `val_lower_bound`
 * (n_val_lanes u64; NULL = no bound) are dropped, keys left without values
 * vanish.  OrdZSet batches (n_val_lanes == 0) ignore the bound
 * (zset_batch.rs:307-318). */
int32_t dbsp_batch_merge_bounded(dbsp_ctx* ctx, const dbsp_batch* a,
                                 const dbsp_batch* b,
                                 const uint64_t* val_lower_bound,
                                 dbsp_batch** out);
/* The fuelled Merger (trace/mod.rs:371-396: new_merger / work / done).
 * work() spends at most *fuel units (here: input rows) and subtracts what it
 * used; *fuel > 0 after the call <=> the merge is complete (:388-395).
 * *fuel <= 0 is not an error: no work is done and *fuel comes back unchanged
 * (as 1 when the merge is already complete).  done() requires a complete
 * merge (else DBSP_ERR_INVALID and the merger stays the caller's), returns
 * the batch and frees the merger.  a and b must have one schema. */
typedef struct dbsp_merger dbsp_merger;
int32_t dbsp_merger_new(dbsp_ctx* ctx, const dbsp_batch* a, const dbsp_batch* b,
                        const uint64_t* val_lower_bound, dbsp_merger** out);
int32_t dbsp_merger_work(dbsp_ctx* ctx, dbsp_merger* m, int64_t* fuel);
int32_t dbsp_merger_done(dbsp_ctx* ctx, dbsp_merger* m, dbsp_batch** out);
int32_t dbsp_merger_free(dbsp_merger* m);
/* BatchReader::truncate_keys_below (trace/mod.rs:227-233;
 * column_layer/mod.rs:316-319): zero-copy suffix view, key = n_key_lanes u64. */
int32_t dbsp_batch_truncate_keys_below(dbsp_ctx* ctx, const dbsp_batch* b,
                                       const uint64_t* key, dbsp_batch** out);
/* neg (column_layer/mod.rs:452-480). */
int32_t dbsp_batch_neg(dbsp_ctx* ctx, const dbsp_batch* a, dbsp_batch** out);
/* Same rows, different key/value split: `index()` (operator/index.rs:128-157)
 * and its inverse are free in the flat column-major layout. */
int32_t dbsp_batch_reindex(dbsp_ctx* ctx, const dbsp_batch* a,
                           uint32_t n_key_lanes, dbsp_batch** out);
/* BatchReader::len / key_count (trace/mod.rs:179-234). */
int32_t dbsp_batch_len(const dbsp_batch* b, uint64_t* n_tuples);
int32_t dbsp_batch_key_count(dbsp_ctx* ctx, const dbsp_batch* b,
                             uint64_t* n_keys);
int32_t dbsp_batch_schema(const dbsp_batch* b, dbsp_schema* out);
/* Canonical vectors of the reference's batch structs.  Any pointer may be
 * NULL (skipped).  keys[l]: n_keys u64 (n_tuples when n_val_lanes == 0);
 * offs: n_keys+1 (only when n_val_lanes > 0); vals[l], diffs: n_tuples. */
int32_t dbsp_batch_download_csr(dbsp_ctx* ctx, const dbsp_batch* b,
                                uint64_t* const* keys, uint64_t* offs,
                                uint64_t* const* vals, int64_t* diffs);
/* Asynchronous read of a batch's flat rows (the output handle of a circuit
 * drained while the next step runs — the reference's OutputHandle is read by
 * the client thread between steps, operator/output.rs:20-75).  _begin queues,
 * on the context's read stream (its own: PCIe is full duplex, uploads are not
 * delayed) and ordered after the work already queued on the compute stream, the copy of lane l (n_tuples u64) into cols[l] and of
 * the weights into diffs (NULL entries are skipped); the destinations should
 * be pinned host memory and must stay valid until _finish, which waits for
 * the copy and releases the handle (and its reference on the batch). */
typedef struct dbsp_download dbsp_download;
int32_t dbsp_batch_download_begin(dbsp_ctx* ctx, const dbsp_batch* b,
                                  uint64_t* const* cols, int64_t* diffs,
                                  dbsp_download** out);
int32_t dbsp_download_finish(dbsp_download* d);
/* Host synchronisation counters: how many times the host waited for a count
 * published by the device (mailbox read-backs) and for how long in total,
 * since the last reset. */
int32_t dbsp_ctx_sync_stats(dbsp_ctx* ctx, uint64_t* n_waits, double* wait_us,
                            int32_t reset);
/* Device pointers of the flat column-major rows (lane l, weights). */
int32_t dbsp_batch_device_columns(const dbsp_batch* b, const uint64_t** cols,
                                  const int64_t** weights);
/* Largest key (first key lane set) of the batch — `fast_forward_keys` +
 * `get_key` as used by watermark_monotonic (watermark.rs:38-45).
 * *valid = 0 when the batch is empty. */
int32_t dbsp_batch_last_key(dbsp_ctx* ctx, const dbsp_batch* b, uint64_t* key,
                            int32_t* valid);
int32_t dbsp_batch_clone(const dbsp_batch* b, dbsp_batch** out);
int32_t dbsp_batch_free(dbsp_batch* b);

/* ---- spine (trace) -------------------------------------------------- */
/* Spine (trace/spine_fueled.rs:107-119): LSM of immutable batches. */
int32_t dbsp_spine_new(dbsp_ctx* ctx, const dbsp_schema* schema,
                       dbsp_spine** out);
/* Trace::insert (spine_fueled.rs:605-634): the batch is shared, not copied. */
int32_t dbsp_spine_insert(dbsp_ctx* ctx, dbsp_spine* s, const dbsp_batch* b);
/* Trace::consolidate (spine_fueled.rs:583-600): merge everything. */
int32_t dbsp_spine_consolidate(dbsp_ctx* ctx, dbsp_spine* s, dbsp_batch** out);
/* truncate_keys_below (spine_fueled.rs:223-233); `key` = n_key_lanes u64. */
int32_t dbsp_spine_truncate_keys_below(dbsp_ctx* ctx, dbsp_spine* s,
                                       const uint64_t* key);
/* Trace::truncate_values_below (trace/mod.rs:150-169; spine_fueled.rs:644-656):
 * the bound only grows and is applied by later merges and by consolidate;
 * values below it are undefined until then (as in the reference). */
int32_t dbsp_spine_truncate_values_below(dbsp_ctx* ctx, dbsp_spine* s,
                                         const uint64_t* val);
/* Trace::exert (trace/mod.rs:104-113; spine_fueled.rs:627-634).  This spine
 * merges eagerly on insert, so no merge is ever in progress; effort buys extra
 * compaction instead: the two newest batches are merged while their combined
 * length fits *effort (decremented by the rows merged). */
int32_t dbsp_spine_exert(dbsp_ctx* ctx, dbsp_spine* s, int64_t* effort);
int32_t dbsp_spine_len(const dbsp_spine* s, uint64_t* n_tuples,
                       uint32_t* n_batches);
int32_t dbsp_spine_free(dbsp_spine* s);

/* Checkpoint / resume of a trace (SURVEY.md §8(f)4): the device-side replacement of the RocksDB-backed
 * PersistentTrace (crates/dbsp/src/trace/persistent/) for snapshots.  One little-endian file: magic "DBSPSPN1",
 * the schema, key / value bounds, effort, then every layer of the spine (spine_fueled.rs:1012-1027: Vacant /
 * Single / Double{InProgress, Complete}) with its batches as flat lanes + weights and, for a merge in progress,
 * the fuel still owed — so a loaded spine resumes the same merge schedule.  The format is shared with the oracle.
 * dbsp_spine_load treats the file as outside input: every field is checked as it is read and before anything is
 * allocated for it (schema, flags, layer count and kinds, which batches a layer may hold, row counts against the
 * bytes left, the fuel owed, no trailing bytes), and the rows of every batch must be ordered, free of duplicate rows
 * and of zero weights; otherwise DBSP_ERR_INVALID, and everything already loaded is freed. */
int32_t dbsp_spine_save(dbsp_ctx* ctx, const dbsp_spine* s, const char* path);
int32_t dbsp_spine_load(dbsp_ctx* ctx, const char* path, dbsp_spine** out);

/* ---- operators ------------------------------------------------------ */
/* JoinTrace::eval (operator/join.rs:732-863), Time = (): delta joined with
 * every batch of the trace, weights multiplied, join_func = proj, result
 * consolidated.  `delta_is_left` != 0: delta rows feed SRC_LVAL and trace
 * rows SRC_RVAL; 0: swapped (the flipped closure of join.rs:279-284). */
int32_t dbsp_join_delta_trace(dbsp_ctx* ctx, const dbsp_batch* delta,
                              const dbsp_spine* trace, const dbsp_proj* proj,
                              int32_t delta_is_left, dbsp_batch** out);
/* Join::eval (join.rs:436-473): stateless batch x batch.  Both joins need
 * equal key lanes (count and types) on the two sides; `proj` may name the key
 * lanes, the left side's value lanes (LVAL) and the right side's (RVAL). */
int32_t dbsp_join_batches(dbsp_ctx* ctx, const dbsp_batch* left,
                          const dbsp_batch* right, const dbsp_proj* proj,
                          dbsp_batch** out);
/* Both joins with a row function as join_func; a row whose keep flag is 0
 * is dropped. */
int32_t dbsp_join_delta_trace_fn(dbsp_ctx* ctx, const dbsp_batch* delta,
                                 const dbsp_spine* trace, const dbsp_rowfn* fn,
                                 int32_t delta_is_left, dbsp_batch** out);
int32_t dbsp_join_batches_fn(dbsp_ctx* ctx, const dbsp_batch* left,
                             const dbsp_batch* right, const dbsp_rowfn* fn,
                             dbsp_batch** out);
/* SemiJoinStream::eval (operator/semijoin.rs:100-142).  `keys` has the key
 * lanes of `pairs` and no value lanes. */
int32_t dbsp_semijoin(dbsp_ctx* ctx, const dbsp_batch* pairs,
                      const dbsp_batch* keys, dbsp_batch** out);
/* AggregateIncremental::eval (aggregate/mod.rs:600-684) fused with
 * Upsert::eval (operator/upsert.rs:161-208): for every key of `delta`,
 * aggregate the key's values in `in_trace` (which already contains delta),
 * compare with the key's current value in `out_trace`, emit -1/+1 rows.
 * The caller then inserts *out into out_trace (the TraceAppend of
 * upsert.rs:69-107).  delta and in_trace have one schema; out_trace has their
 * key lanes (WCOUNT2: all but the last) and the values of the aggregator:
 * MAX / MIN the input's values (at least one lane), FOLD_* one lane over an
 * input with values, WCOUNT one lane and WCOUNT2 two over an input without. */
int32_t dbsp_aggregate_delta(dbsp_ctx* ctx, const dbsp_batch* delta,
                             const dbsp_spine* in_trace,
                             const dbsp_spine* out_trace, int32_t agg_kind,
                             dbsp_batch** out);
/* The same AggregateIncremental + Upsert with a Fold (fold.rs:60-75) as the
 * aggregator.  For every key of `delta`, the key's values in `in_trace` are
 * taken in value order with their weights summed over the batches, and values
 * whose sum is 0 are skipped.  Starting from fold->init, `step` runs once per
 * remaining value, serially (Fold is not associative).  A key with at least
 * one such value gets the row (key, output(acc)) unless output's keep flag is
 * 0; a key with none gets no row.  The result is -old +new against
 * `out_trace`, as in dbsp_aggregate_delta.  delta and in_trace have one
 * schema; out_trace has delta's key lanes followed by fold->output's value
 * lanes (count and types). */
int32_t dbsp_aggregate_fold(dbsp_ctx* ctx, const dbsp_batch* delta,
                            const dbsp_spine* in_trace,
                            const dbsp_spine* out_trace, const dbsp_fold* fold,
                            dbsp_batch** out);
/* The commands of a set or map input table (operator/input.rs:128-328,
 * add_input_set / add_input_map) as a batch.  `table` is the table's schema:
 * at least one key lane and at most 7 lanes in all (a set has key lanes
 * only).  The batch has the table's key lanes as its keys, then as values one
 * u64 command lane and the table's value lanes.  Command i (0 <= i < n) is
 * the row cols[0..nk+nv)[i] with the command word
 *   ((seq0 + i) << 1) | (insert[i] != 0)
 * and weight 1; a delete's value lanes are written as 0.  insert == NULL:
 * every command inserts.  seq0 + n is at most 2^63 (a sequence number has 63
 * bits).  on_device as in dbsp_batch_from_tuples (cols and insert).  The rows are
 * consolidated, so they come out ordered by (key, command word): a stable sort
 * by key of the commands in sequence order (input.rs:141-145).  Batches of
 * commands with distinct sequence numbers merge (and shard) into one batch in
 * the same order. */
int32_t dbsp_upsert_commands(dbsp_ctx* ctx, const dbsp_schema* table,
                             const uint64_t* const* cols,
                             const uint8_t* insert, uint64_t n, uint64_t seq0,
                             int32_t on_device, dbsp_batch** out);
/* Upsert::eval (operator/upsert.rs:155-208) of a command batch against the
 * table's trace: per key with a command, only the last command counts
 * (input.rs:147-160); the key's current rows in `table` (weights summed over
 * its batches, zero sums skipped) are retracted with their negated weights,
 * and (key, v) is inserted with weight +1 if that command inserts.  The
 * result is consolidated, with the table's schema; the caller inserts it into
 * `table` (upsert.rs:69-107).  `cmds` has the schema dbsp_upsert_commands
 * gives for the table; its weights are not read. */
int32_t dbsp_upsert_delta(dbsp_ctx* ctx, const dbsp_batch* cmds,
                          const dbsp_spine* table, dbsp_batch** out);
/* Relative time range of a rolling aggregate (time_series/range.rs RelRange /
 * RelOffset).  Each end is Before(off) or After(off), off a magnitude.  For a
 * timestamp ts, range_of(ts) = [from(ts), to(ts)] in the TS lane's type: a
 * `from` Before saturates and After is a checked add (overflow: no range); a
 * `to` Before is a checked subtract (underflow: no range) and After saturates.
 * affected_range_of(ts), the times whose range holds ts, mirrors it. */
typedef struct dbsp_rel_range {
  uint8_t from_after, to_after;   /* 0 = Before(off), 1 = After(off) */
  uint8_t pad_[6];
  uint64_t from_off, to_off;      /* magnitudes; i64 TS: at most INT64_MAX */
} dbsp_rel_range;
enum dbsp_rolling_kind { DBSP_ROLLING_LINEAR = 0, DBSP_ROLLING_MAX = 1, DBSP_ROLLING_MIN = 2 };
/* PartitionedRollingAggregate::eval (time_series/rolling_aggregate.rs:436-604).
 * delta and in_trace have one schema: the key lanes are the partition key PK
 * (none: one partition), value lane 0 is the timestamp TS and the other value
 * lanes are V.  For every (pk, ts) with a row of positive weight in in_trace
 * (weights summed over its batches) and a range_of(ts), the output integral
 * holds (pk, (ts, some, agg..)) with weight 1, where agg aggregates the rows
 * (pk, ts', v) of non-zero weight with ts' in range_of(ts):
 *   LINEAR  per output lane of f(pk, v) (a dbsp_rowfn over KEY, LVAL = V and
 *           CONST with value lanes only), the sum of f * weight, wrapping;
 *           a row whose keep flag is 0 adds 0;
 *   MAX/MIN the lexicographically greatest / least V tuple (max.rs:36-55).
 * some = 0 (and agg lanes 0) when no row lies in the range.  The call returns
 * the change of that integral for the times the delta affects (the union of
 * affected_range_of(d) and [d, d] per delta time d): out_trace's rows there
 * retracted, the recomputed rows inserted.  out_trace has PK's key lanes and
 * the value lanes (TS, u64 some, agg lanes): f's lanes or V's.  As with
 * dbsp_aggregate_delta, the caller has already inserted delta into in_trace
 * and inserts *out into out_trace afterwards; in_trace need not be delta's
 * integral (the watermark form feeds it a windowed stream).  `f` is given for
 * LINEAR and must be NULL otherwise.  A delta of 2^30 or more rows, or 16
 * trace batches of 2^32-1 or more rows, is DBSP_ERR_UNSUPPORTED. */
int32_t dbsp_rolling_aggregate(dbsp_ctx* ctx, const dbsp_batch* delta, const dbsp_spine* in_trace,
                               const dbsp_spine* out_trace, const dbsp_rel_range* range, int32_t kind,
                               const dbsp_rowfn* f, dbsp_batch** out);
/* weigh (aggregate/mod.rs:297-323). `f` gives f(k,v) (SRC_KEY/SRC_LVAL).
 * `mode` is a dbsp_weigh_mode; WEIGH_AVG adds a key lane (at most 7 before). */
int32_t dbsp_weigh(dbsp_ctx* ctx, const dbsp_batch* b, const dbsp_expr* f,
                   int32_t mode, dbsp_batch** out);
/* weigh with a row function: fn->out_schema has one lane, the factor f(k,v);
 * a row whose keep flag is 0 contributes nothing (in WEIGH_AVG mode neither
 * to the sum nor to the count). */
int32_t dbsp_weigh_fn(dbsp_ctx* ctx, const dbsp_batch* b, const dbsp_rowfn* fn,
                      int32_t mode, dbsp_batch** out);
/* DistinctIncrementalTotal::eval (operator/distinct.rs:196-254).  delta and
 * the integral have one schema. */
int32_t dbsp_distinct_delta(dbsp_ctx* ctx, const dbsp_batch* delta,
                            const dbsp_spine* delayed_integral,
                            dbsp_batch** out);
/* The change of antijoin (operator/join.rs:294-320) without expanding a key's
 * values.  With N(k) the number of distinct (k, v2) rows of the other side
 * (the rows of distinct(other) on key k), the antijoin gives a row (k, v1, w)
 * the weight w·(1 − N(k)), wrapping; so its change is
 *   out = delta·(1 − key_trace(k)) − trace ⋉ key_delta,
 * consolidated, with delta's schema.  `trace` is z^-1 of delta's integral
 * (delta's schema).  `key_delta` and `key_trace` are OrdZSet<K>s with exactly
 * delta's key lanes (count and types) and no value lanes: a row's weight is
 * the change of its key's count (key_delta) or the count itself (key_trace,
 * which already includes key_delta; key_trace(k) sums k's weights over its
 * batches).  delta has at least one key lane. */
int32_t dbsp_antijoin_delta(dbsp_ctx* ctx, const dbsp_batch* delta,
                            const dbsp_spine* trace, const dbsp_batch* key_delta,
                            const dbsp_spine* key_trace, dbsp_batch** out);
/* IndexedZSet::distinct (algebra/zset/mod.rs:14-38). */
int32_t dbsp_stream_distinct(dbsp_ctx* ctx, const dbsp_batch* b,
                             dbsp_batch** out);
/* Window::eval (operator/time_series/window.rs:144-222).  Bounds are
 * n_key_lanes u64 each; has_prev == 0 on the first step (start0 / end0 may
 * then be NULL).  trace and delta have one schema. */
int32_t dbsp_window_delta(dbsp_ctx* ctx, const dbsp_spine* trace,
                          const dbsp_batch* delta, int32_t has_prev,
                          const uint64_t* start0, const uint64_t* end0,
                          const uint64_t* start1, const uint64_t* end1,
                          dbsp_batch** out);
/* Map/FlatMap/Index::eval + from_tuples (filter_map.rs:563-577,700-724). */
int32_t dbsp_map_index(dbsp_ctx* ctx, const dbsp_batch* b,
                       const dbsp_proj* proj, dbsp_batch** out);
int32_t dbsp_map_index_fn(dbsp_ctx* ctx, const dbsp_batch* b,
                          const dbsp_rowfn* fn, dbsp_batch** out);
/* flat_map / flat_map_index of a batch with a fan-out (see
 * dbsp_batch_from_table_fanout): n_out runs of fn per row, j pushed by
 * DBSP_SRC_FANOUT. */
int32_t dbsp_map_index_fanout(dbsp_ctx* ctx, const dbsp_batch* b,
                              const dbsp_rowfn* fn, uint32_t n_out,
                              dbsp_batch** out);
/* shard_batch (operator/communication/shard.rs:165-199): split by
 * hash(key) % n_shards into n_shards (1..64) ordered batches.  The exchange itself
 * (exchange.rs:128-200) is done by the host with its collective library on
 * dbsp_batch_device_columns(); the receiver merges (shard.rs:136-144). */
int32_t dbsp_shard_partition(dbsp_ctx* ctx, const dbsp_batch* b,
                             uint32_t n_shards, dbsp_batch** outs);
/* ---- communication between circuit replicas (one replica = one context = one GPU) ----------------
 * Replaces shard (operator/communication/shard.rs:106-162), Exchange (exchange.rs:128-200), gather
 * (gather.rs:41-103) and the watermark exchange (time_series/watermark.rs:53-70) — the three calls SURVEY.md
 * §8(b) lists as dbsp_shard / dbsp_gather / dbsp_allreduce_max_u64.  There is no collective library on the
 * data path: every context owns a device receive region; peers map it (CUDA IPC between processes, peer
 * access between the contexts of one process) and the partition kernel's stores land in it over NVLink.
 *
 * Bootstrap (replaces the ncclUniqueId of the survey's sketch): every rank calls dbsp_comm_create, which
 * returns a DBSP_COMM_BLOB_BYTES descriptor of its region; the HOST moves the `world` descriptors to every
 * rank by whatever channel it has (the reference's workers are threads of one process: a shared Vec; one
 * process per GPU: any all-gather) and hands the rank-ordered array to dbsp_comm_connect.
 * All replicas must issue the same sequence of exchange calls (they run the same circuit). */
#define DBSP_COMM_MAX_RANKS 32
#define DBSP_COMM_BLOB_BYTES 128
int32_t dbsp_comm_create(dbsp_ctx* ctx, int32_t rank, int32_t world,
                         uint64_t slot_bytes /* capacity of one (source,destination) segment per round; 0 = 512 MiB */,
                         uint8_t* blob_out /* DBSP_COMM_BLOB_BYTES */);
int32_t dbsp_comm_connect(dbsp_ctx* ctx, const uint8_t* blobs /* world * DBSP_COMM_BLOB_BYTES, rank order */);
int32_t dbsp_comm_destroy(dbsp_ctx* ctx);
/* rank / world of the context (0 / 1 without a comm) and payload bytes it has sent to other ranks */
int32_t dbsp_comm_info(dbsp_ctx* ctx, int32_t* rank, int32_t* world, uint64_t* bytes_sent);
/* Stream::shard (shard.rs:106-162): rows re-partitioned by hash(key) % world; returns this replica's shard,
 * consolidated (partition + NVLink scatter + receiver merge in one call; identity when world == 1). */
int32_t dbsp_shard(dbsp_ctx* ctx, const dbsp_batch* b, dbsp_batch** out);
/* shard() of both inputs of a binary operator (join.rs:265-266) in ONE exchange round. */
int32_t dbsp_shard2(dbsp_ctx* ctx, const dbsp_batch* a, const dbsp_batch* b,
                    dbsp_batch** out_a, dbsp_batch** out_b);
/* Stream::gather (gather.rs:41-103): everything to `root`, empty batches elsewhere. */
int32_t dbsp_gather(dbsp_ctx* ctx, const dbsp_batch* b, int32_t root, dbsp_batch** out);
/* max over the replicas of *x (watermark.rs:53-70); every replica gets the result. */
int32_t dbsp_allreduce_max_u64(dbsp_ctx* ctx, uint64_t* x);

/* Builder path (trace/mod.rs:338-368): adopt rows that are already sorted
 * and consolidated (e.g. a segment received from a peer).  `weights` is
 * required; the rows are taken on trust. */
int32_t dbsp_batch_from_sorted(dbsp_ctx* ctx, const dbsp_schema* schema,
                               const uint64_t* const* cols,
                               const int64_t* weights, uint64_t n,
                               int32_t on_device, dbsp_batch** out);

#ifdef __cplusplus
}
#endif
#endif /* DBSP_B200_H */
