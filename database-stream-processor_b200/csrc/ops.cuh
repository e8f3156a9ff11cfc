// ops.cuh — host entry points of the operator kernels (ops.cu).
#pragma once
#include <algorithm>
#include <cstring>
#include <type_traits>

#include "common.cuh"

int32_t compact_ordered(Ctx* ctx, const dbsp_schema& s, const Cols& in, const i64* w, const u32* keep, u64 n, Batch** out);
unsigned proj_used_mask(const dbsp_proj& p, int nk_in);
unsigned rowfn_used_mask(const dbsp_rowfn& f, int nk_in);
// A row function run n_out times per input row (the `_fanout` calls): a third closure form of the projection, whose
// program may push DBSP_SRC_FANOUT.  It is a dbsp_rowfn, so every helper of row functions takes it as one.
struct RowFnFanout : dbsp_rowfn {
  u32 n_out;
};
// The closure-taking operators, for F = dbsp_proj and F = dbsp_rowfn (weigh: dbsp_expr and dbsp_rowfn); the
// projection (project_and_consolidate, op_map_index) also for F = RowFnFanout.
template <class F>
int32_t project_and_consolidate(Ctx* ctx, const Cols& in, int nk_in, int n_in_lanes, const i64* w, u64 n,
                                const F& proj, Batch** out);
template <class F>
int32_t op_join_delta_trace(Ctx* ctx, const Batch* delta, const Spine* trace, const F* proj, int delta_is_left,
                            Batch** out);
template <class F>
int32_t op_join_batches(Ctx* ctx, const Batch* l, const Batch* r, const F* proj, Batch** out);
int32_t op_aggregate_delta(Ctx* ctx, const Batch* delta, const Spine* in_tr, const Spine* out_tr, int kind, Batch** out);
int32_t op_aggregate_fold(Ctx* ctx, const Batch* delta, const Spine* in_tr, const Spine* out_tr, const dbsp_fold* fold,
                          Batch** out);
int32_t op_rolling_aggregate(Ctx* ctx, const Batch* delta, const Spine* in_tr, const Spine* out_tr,
                             const dbsp_rel_range& range, int kind, const dbsp_rowfn* f, Batch** out);
int32_t op_upsert_commands(Ctx* ctx, const dbsp_schema& table, const Cols& in, const uint8_t* insert, u64 n, u64 seq0,
                           Batch** out);
int32_t op_upsert_delta(Ctx* ctx, const Batch* cmds, const Spine* table, Batch** out);
int32_t op_neg(Ctx* ctx, const Batch* a, Batch** out);
template <class F>
int32_t op_weigh(Ctx* ctx, const Batch* b, const F* f, int mode, Batch** out);
int32_t op_distinct_delta(Ctx* ctx, const Batch* delta, const Spine* integral, Batch** out);
int32_t op_antijoin_delta(Ctx* ctx, const Batch* delta, const Spine* trace, const Batch* key_delta,
                          const Spine* key_trace, Batch** out);
int32_t op_stream_distinct(Ctx* ctx, const Batch* b, Batch** out);
int32_t op_semijoin(Ctx* ctx, const Batch* pairs, const Batch* keys, Batch** out);
int32_t op_window_delta(Ctx* ctx, const Spine* trace, const Batch* delta, int has_prev, const u64* s0, const u64* e0,
                        const u64* s1, const u64* e1, Batch** out);
template <class F>
int32_t op_map_index(Ctx* ctx, const Batch* b, const F* proj, Batch** out);
int32_t op_shard_partition(Ctx* ctx, const Batch* b, u32 P, Batch** outs);
int32_t batch_build_csr(Ctx* ctx, Batch* b);
int32_t batch_lower_bound(Ctx* ctx, const Batch* b, const u64* key, u64* pos);
int32_t op_truncate_values(Ctx* ctx, const Batch* b, const u64* val_bound, Batch** out);
Batch* batch_slice(Ctx* ctx, const Batch* b, u64 lo, u64 hi);
int32_t batch_concat(Ctx* ctx, const dbsp_schema& s, std::vector<Batch*>& parts, Batch** out);
