// validate.h — the argument and snapshot-file rules of the C ABI (include/dbsp_b200.h "Error contract").
//
// Plain C++, no CUDA types: the CUDA library (capi.cu) and the CPU oracle (oracle/dbsp_oracle.cpp) refuse the same
// inputs with the same texts.  Validation is not an algorithm; the oracle's independence is about the operators.
// Every check is O(1) in the row count.  A function returns the empty string when the argument is acceptable and
// otherwise the text for dbsp_last_error, which names the call (`what`) and the argument.
#pragma once
#include <stdint.h>

#include <string>

#include "../../include/dbsp_b200.h"

namespace dbsp_validate {

inline std::string num(uint64_t v) { return std::to_string(v); }

// 1..8 lanes in total (counted without wrapping), every lane u64 or i64
inline std::string valid_schema(const dbsp_schema* s, const std::string& what, const char* arg = "schema") {
  if (!s) return what + ": " + arg + " is NULL";
  const int L = (int)s->n_key_lanes + (int)s->n_val_lanes;
  if (L < 1 || L > DBSP_MAX_LANES)
    return what + ": " + arg + " must have 1..8 lanes, has " + num(s->n_key_lanes) + " key + " + num(s->n_val_lanes) + " value lanes";
  for (int l = 0; l < L; l++)
    if (s->lane_types[l] > DBSP_I64) return what + ": " + arg + ".lane_types[" + num(l) + "] = " + num(s->lane_types[l]) + " is not a lane type";
  return "";
}

inline bool same_key_lanes(const dbsp_schema& a, const dbsp_schema& b) {
  if (a.n_key_lanes != b.n_key_lanes) return false;
  for (int l = 0; l < a.n_key_lanes; l++)
    if (a.lane_types[l] != b.lane_types[l]) return false;
  return true;
}
inline bool same_schema(const dbsp_schema& a, const dbsp_schema& b) {
  if (a.n_key_lanes != b.n_key_lanes || a.n_val_lanes != b.n_val_lanes) return false;
  for (int l = 0; l < a.n_key_lanes + a.n_val_lanes; l++)
    if (a.lane_types[l] != b.lane_types[l]) return false;
  return true;
}

// A source may name lane idx < nk of the key, < n_lval of the left value, < n_rval of the right value.  Calls with
// one input (map_index, weigh, raw tables) pass n_rval = n_lval: there SRC_RVAL reads the same lanes as SRC_LVAL.
inline std::string valid_src(const dbsp_src& s, int nk, int n_lval, int n_rval, const std::string& where) {
  static const char* const names[] = {"SRC_KEY", "SRC_LVAL", "SRC_RVAL"};
  if (s.kind > DBSP_SRC_CONST) return where + ".kind = " + num(s.kind) + " is not a source kind";
  if (s.kind == DBSP_SRC_CONST) return "";
  const int have = s.kind == DBSP_SRC_KEY ? nk : s.kind == DBSP_SRC_LVAL ? n_lval : n_rval;
  if (s.idx >= have) return where + ".idx = " + num(s.idx) + ": " + names[s.kind] + " has " + num(have) + " lanes";
  return "";
}
inline std::string valid_expr(const dbsp_expr* e, int nk, int n_lval, int n_rval, const std::string& where) {
  if (!e) return where + " is NULL";
  if (e->op > DBSP_OP_DIV) return where + ".op = " + num(e->op) + " is not an operation";
  std::string m = valid_src(e->a, nk, n_lval, n_rval, where + ".a");
  if (m.empty() && e->op >= DBSP_OP_ADD) m = valid_src(e->b, nk, n_lval, n_rval, where + ".b");
  return m;
}
inline std::string valid_proj(const dbsp_proj* p, int nk, int n_lval, int n_rval, const std::string& what) {
  if (!p) return what + ": proj is NULL";
  std::string m = valid_schema(&p->out_schema, what, "proj.out_schema");
  if (!m.empty()) return m;
  if (p->n_pred > DBSP_MAX_PREDS) return what + ": proj.n_pred = " + num(p->n_pred) + " exceeds " + num(DBSP_MAX_PREDS);
  const int L = p->out_schema.n_key_lanes + p->out_schema.n_val_lanes;
  for (int l = 0; l < L; l++) {
    m = valid_expr(&p->out[l], nk, n_lval, n_rval, what + ": proj.out[" + num(l) + "]");
    if (!m.empty()) return m;
  }
  for (int i = 0; i < p->n_pred; i++) {
    const std::string where = what + ": proj.pred[" + num(i) + "]";
    if (p->pred[i].cmp > DBSP_CMP_IN) return where + ".cmp = " + num(p->pred[i].cmp) + " is not a comparison";
    m = valid_src(p->pred[i].a, nk, n_lval, n_rval, where + ".a");
    if (m.empty()) m = valid_src(p->pred[i].b, nk, n_lval, n_rval, where + ".b");
    if (!m.empty()) return m;
  }
  return "";
}
// columns of a raw table a projection reads (bit l = column l); call after valid_proj
inline uint32_t proj_table_mask(const dbsp_proj& p) {
  uint32_t mask = 0;
  auto use = [&](const dbsp_src& s) { if (s.kind != DBSP_SRC_CONST) mask |= 1u << s.idx; };
  const int L = p.out_schema.n_key_lanes + p.out_schema.n_val_lanes;
  for (int l = 0; l < L; l++) { use(p.out[l].a); if (p.out[l].op >= DBSP_OP_ADD) use(p.out[l].b); }
  for (int i = 0; i < p.n_pred; i++) { use(p.pred[i].a); use(p.pred[i].b); }
  return mask;
}

// What an aggregate needs of its three operands: delta and the input trace share one schema, the output trace has
// their key lanes, and each kind its own value shape.
inline std::string valid_aggregate(const dbsp_schema& delta, const dbsp_schema& in, const dbsp_schema& out, int32_t kind) {
  const std::string what = "aggregate_delta";
  if (kind < DBSP_AGG_MAX || kind > DBSP_AGG_WCOUNT2) return what + ": agg_kind = " + std::to_string(kind) + " is not an aggregator";
  if (!same_schema(delta, in)) return what + ": delta and in_trace differ in schema";
  const int nv = in.n_val_lanes;
  if (kind == DBSP_AGG_WCOUNT2) {   // delta rows are (K.., which): the output key is all but the last key lane
    if (nv != 0 || out.n_key_lanes != in.n_key_lanes - 1 || out.n_val_lanes != 2)
      return what + ": AGG_WCOUNT2 needs delta (K.., which) without values and out_trace (K..) -> (sum, count)";
    for (int l = 0; l < out.n_key_lanes; l++)
      if (out.lane_types[l] != in.lane_types[l]) return what + ": delta and out_trace differ in key lane types";
    return "";
  }
  if (!same_key_lanes(delta, out)) return what + ": delta and out_trace differ in key lanes";
  if (kind == DBSP_AGG_MAX || kind == DBSP_AGG_MIN) {
    if (nv == 0 || out.n_val_lanes != nv) return what + ": AGG_MAX / AGG_MIN need out_trace values shaped like in_trace values (at least one lane)";
    for (int l = 0; l < nv; l++)
      if (out.lane_types[out.n_key_lanes + l] != in.lane_types[in.n_key_lanes + l]) return what + ": in_trace and out_trace differ in value lane types";
    return "";
  }
  if (out.n_val_lanes != 1) return what + ": this agg_kind writes one value lane to out_trace";
  if (kind == DBSP_AGG_WCOUNT ? nv != 0 : nv == 0)
    return what + (kind == DBSP_AGG_WCOUNT ? ": AGG_WCOUNT needs a delta without value lanes" : ": AGG_FOLD_* need a delta with value lanes");
  return "";
}

// ---- snapshot files (dbsp_spine_save / dbsp_spine_load) ---------------------------------------------------------
// header: magic, schema, {has key bound, has value bound, effort, layer count}, key bound, value bound
inline std::string valid_snapshot_header(const dbsp_schema& s, const uint64_t hdr[4]) {
  std::string m = valid_schema(&s, "spine_load", "file schema");
  if (!m.empty()) return m;
  if (hdr[0] > 1 || hdr[1] > 1) return "spine_load: bound flag " + num(hdr[0] > 1 ? hdr[0] : hdr[1]) + " is neither 0 nor 1";
  if (hdr[3] > 64) return "spine_load: layer count " + num(hdr[3]) + " exceeds 64";
  return "";
}
enum { SNAP_VACANT = 0, SNAP_SINGLE = 1, SNAP_IN_PROGRESS = 2, SNAP_COMPLETE = 3 };
inline std::string valid_snapshot_kind(uint64_t kind) {
  return kind > SNAP_COMPLETE ? "spine_load: layer kind " + num(kind) + " is not a layer state" : "";
}
// the header of batch `which` (0 = a, 1 = b) of a layer, before anything is allocated for it.  A vacant layer holds
// nothing, a merge in progress both inputs, a single or complete layer at most `a` (exert leaves layers that are
// structurally occupied and hold no batch).
inline std::string valid_snapshot_batch(uint64_t kind, int which, uint64_t present, uint64_t n, int lanes, uint64_t bytes_left) {
  const char* name = which ? "b" : "a";
  if (present > 1) return std::string("spine_load: presence of batch ") + name + " = " + num(present) + " is neither 0 nor 1";
  const bool required = kind == SNAP_IN_PROGRESS, allowed = required || (which == 0 && kind != SNAP_VACANT);
  if (present && !allowed) return std::string("spine_load: layer kind ") + num(kind) + " cannot hold batch " + name;
  if (!present && required) return std::string("spine_load: merge in progress without batch ") + name;
  if (!present && n) return std::string("spine_load: absent batch ") + name + " with " + num(n) + " rows";
  if (n >= (1ull << 32)) return std::string("spine_load: batch ") + name + " has 2^32 or more rows";
  if (n * 8 * (uint64_t)(lanes + 1) > bytes_left) return std::string("spine_load: truncated file (batch ") + name + " of " + num(n) + " rows does not fit)";
  return "";
}
inline std::string valid_snapshot_remaining(uint64_t remaining, uint64_t len_a, uint64_t len_b) {
  if ((int64_t)remaining < 0 || remaining > len_a + len_b) return "spine_load: remaining fuel " + std::to_string((int64_t)remaining) + " outside 0.." + num(len_a + len_b);
  return "";
}

}  // namespace dbsp_validate
