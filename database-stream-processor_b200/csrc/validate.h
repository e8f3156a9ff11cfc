// validate.h — the argument and snapshot-file rules of the C ABI (include/dbsp_b200.h "Error contract").
//
// Plain C++, no CUDA types: the CUDA library (capi.cu) and the CPU oracle (oracle/dbsp_oracle.cpp) refuse the same
// inputs with the same texts.  Validation is not an algorithm; the oracle's independence is about the operators.
// Every check is O(1) in the row count.  A function returns the empty string when the argument is acceptable and
// otherwise the text for dbsp_last_error, which names the call (`what`) and the argument.
#pragma once
#include <stdint.h>
#include <string.h>

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

// Operands an instruction pops (it pushes one value; PUSH pops none)
inline int rowfn_arity(uint8_t op) {
  if (op == DBSP_FN_PUSH) return 0;
  if (op <= DBSP_FN_LNOT) return 1;
  return op == DBSP_FN_SELECT ? 3 : 2;
}
// The source kinds beyond KEY / LVAL / RVAL / CONST a call lets a PUSH take (valid_rowfn's `extra`)
constexpr unsigned SRC_BIT_FANOUT = 1u << DBSP_SRC_FANOUT, SRC_BIT_ACC = 1u << DBSP_SRC_ACC,
                   SRC_BIT_WEIGHT = 1u << DBSP_SRC_WEIGHT;
// A row function: the instructions fit the array, every op and PUSH source is valid for the call (lanes as in
// valid_src), the stack never underflows or exceeds DBSP_MAX_STACK, and it ends with the output lanes + the keep flag.
// One pass over the program, so the depth at each instruction is known before any row is evaluated.  `extra`: the
// further source kinds a PUSH may take (SRC_BIT_*): DBSP_SRC_FANOUT in a `_fanout` call (j; idx and cst ignored),
// DBSP_SRC_ACC (word idx < n_acc) and DBSP_SRC_WEIGHT (idx and cst ignored) in a fold's programs.  `end` >= 0: the
// depth the program must end with instead (a fold's step: its n_acc words + the keep flag).  `arg` names the program.
inline std::string valid_rowfn(const dbsp_rowfn* f, int nk, int n_lval, int n_rval, const std::string& what,
                               unsigned extra = 0, int n_acc = 0, int end = -1, const std::string& arg = "fn") {
  if (!f) return what + ": " + arg + " is NULL";
  std::string m = valid_schema(&f->out_schema, what, (arg + ".out_schema").c_str());
  if (!m.empty()) return m;
  if (f->n_insn > DBSP_MAX_INSNS) return what + ": " + arg + ".n_insn = " + num(f->n_insn) + " exceeds " + num(DBSP_MAX_INSNS);
  int depth = 0;
  for (int i = 0; i < f->n_insn; i++) {
    const dbsp_insn& in = f->code[i];
    const std::string where = what + ": " + arg + ".code[" + num(i) + "]";
    if (in.op > DBSP_FN_SELECT) return where + ".op = " + num(in.op) + " is not an instruction";
    const bool allowed = in.kind < 32 && ((extra >> in.kind) & 1);
    if (in.op == DBSP_FN_PUSH && allowed && in.kind == DBSP_SRC_ACC && in.idx >= n_acc)
      return where + ".idx = " + num(in.idx) + ": SRC_ACC has " + num(n_acc) + " words";
    if (in.op == DBSP_FN_PUSH && !allowed) {
      dbsp_src s;
      s.kind = in.kind;
      s.idx = in.idx;
      s.cst = in.cst;
      m = valid_src(s, nk, n_lval, n_rval, where);
      if (!m.empty()) return m;
    }
    const int pops = rowfn_arity(in.op);
    if (depth < pops) return where + ": stack underflow (depth " + num(depth) + ", the op takes " + num(pops) + ")";
    depth += 1 - pops;
    if (depth > DBSP_MAX_STACK) return where + ": stack deeper than " + num(DBSP_MAX_STACK);
  }
  const int L = f->out_schema.n_key_lanes + f->out_schema.n_val_lanes;
  if (end >= 0 && depth != end)
    return what + ": " + arg + " ends with stack depth " + num(depth) + ", needs " + num(end) + " (the accumulator words, then the keep flag)";
  if (end < 0 && depth != L + 1)
    return what + ": " + arg + " ends with stack depth " + num(depth) + ", needs " + num(L + 1) + " (the output lanes, then the keep flag)";
  return "";
}
// columns of a raw table a row function reads (bit l = column l); call after valid_rowfn
inline uint32_t rowfn_table_mask(const dbsp_rowfn& f) {
  uint32_t mask = 0;
  for (int i = 0; i < f.n_insn; i++)
    if (f.code[i].op == DBSP_FN_PUSH && f.code[i].kind < DBSP_SRC_CONST) mask |= 1u << f.code[i].idx;
  return mask;
}
// A fan-out's output count: 1..DBSP_MAX_FANOUT runs of the program per input row
inline std::string valid_fanout(uint32_t n_out, const std::string& what) {
  if (n_out < 1 || n_out > DBSP_MAX_FANOUT)
    return what + ": n_out = " + num(n_out) + ": a fan-out gives 1.." + num(DBSP_MAX_FANOUT) + " rows per input row";
  return "";
}
// n input rows fanned out to n * n_out rows before consolidation: row indices are 32-bit on the device, so 2^32-1 or
// more is refused (DBSP_ERR_UNSUPPORTED), from the sizes alone.  n < 2^32 and n_out <= 64: the product cannot wrap.
inline std::string valid_fanout_rows(uint64_t n, uint32_t n_out, const std::string& what) {
  if (n * (uint64_t)n_out >= 0xffffffffull)
    return what + ": n * n_out = " + num(n) + " * " + num(n_out) + ": 2^32-1 or more rows before consolidation; split the input";
  return "";
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

// A fold's step as a dbsp_rowfn (its code, and a one-lane out_schema that only valid_schema reads: the step's end
// depth is n_acc + 1, given to valid_rowfn as `end`), so that one validator and one interpreter run both programs.
// Call with n_step <= DBSP_MAX_INSNS.
inline dbsp_rowfn fold_step_rowfn(const dbsp_fold& f) {
  dbsp_rowfn r;
  memset(&r, 0, sizeof(r));
  r.out_schema.n_val_lanes = 1;
  r.n_insn = f.n_step;
  memcpy(r.code, f.step, sizeof(dbsp_insn) * f.n_step);
  return r;
}

// aggregate_fold: what aggregate_delta needs of delta / in_trace, the two programs, and an out_trace of delta's key
// lanes followed by exactly the output program's value lanes.
inline std::string valid_fold(const dbsp_schema& delta, const dbsp_schema& in, const dbsp_schema& out, const dbsp_fold* f) {
  const std::string what = "aggregate_fold";
  if (!f) return what + ": fold is NULL";
  if (f->n_acc < 1 || f->n_acc > DBSP_MAX_ACC)
    return what + ": fold.n_acc = " + num(f->n_acc) + ": an accumulator has 1.." + num(DBSP_MAX_ACC) + " words";
  if (f->n_step > DBSP_MAX_INSNS) return what + ": fold.n_step = " + num(f->n_step) + " exceeds " + num(DBSP_MAX_INSNS);
  const dbsp_rowfn step = fold_step_rowfn(*f);
  std::string m = valid_rowfn(&step, delta.n_key_lanes, delta.n_val_lanes, delta.n_val_lanes, what,
                              SRC_BIT_ACC | SRC_BIT_WEIGHT, f->n_acc, f->n_acc + 1, "fold.step");
  if (!m.empty()) return m;
  m = valid_rowfn(&f->output, delta.n_key_lanes, 0, 0, what, SRC_BIT_ACC, f->n_acc, -1, "fold.output");
  if (!m.empty()) return m;
  const dbsp_schema& os = f->output.out_schema;
  if (os.n_key_lanes != 0) return what + ": fold.output.out_schema has key lanes; the output is the key's value lanes only";
  if (!same_schema(delta, in)) return what + ": delta and in_trace differ in schema";
  if (!same_key_lanes(delta, out)) return what + ": delta and out_trace differ in key lanes";
  if (out.n_val_lanes != os.n_val_lanes) return what + ": out_trace must have fold.output's value lanes (count and type)";
  for (int l = 0; l < os.n_val_lanes; l++)
    if (out.lane_types[out.n_key_lanes + l] != os.lane_types[l])
      return what + ": out_trace must have fold.output's value lanes (count and type)";
  return "";
}

// antijoin_delta: delta and trace share one schema with at least one key lane (a key-less stream has no key set to
// count); key_delta and key_trace have exactly delta's key lanes and no value lanes.
inline std::string valid_antijoin(const dbsp_schema& delta, const dbsp_schema& trace, const dbsp_schema& key_delta,
                                  const dbsp_schema& key_trace) {
  const std::string what = "antijoin_delta";
  if (!same_schema(delta, trace)) return what + ": delta and trace differ in schema";
  if (delta.n_key_lanes == 0) return what + ": delta has no key lanes, so there is no key set to count";
  if (!same_key_lanes(delta, key_delta) || key_delta.n_val_lanes != 0)
    return what + ": key_delta must have exactly delta's key lanes (count and type) and no value lanes";
  if (!same_key_lanes(delta, key_trace) || key_trace.n_val_lanes != 0)
    return what + ": key_trace must have exactly delta's key lanes (count and type) and no value lanes";
  return "";
}

// ---- set and map input tables (dbsp_upsert_commands / dbsp_upsert_delta) ----------------------------------------
// The command batch of a table: its key lanes as keys, then one u64 command lane and its value lanes as values.
inline dbsp_schema upsert_command_schema(const dbsp_schema& t) {
  dbsp_schema c;
  memset(&c, 0, sizeof(c));
  c.n_key_lanes = t.n_key_lanes;
  c.n_val_lanes = (uint8_t)(t.n_val_lanes + 1);
  for (int l = 0; l < t.n_key_lanes; l++) c.lane_types[l] = t.lane_types[l];
  c.lane_types[t.n_key_lanes] = DBSP_U64;
  for (int l = 0; l < t.n_val_lanes; l++) c.lane_types[t.n_key_lanes + 1 + l] = t.lane_types[t.n_key_lanes + l];
  return c;
}
// A table has at least one key lane (an upsert replaces a key's value) and at most 7 lanes (the command lane takes the
// 8th of the command batch).
inline std::string valid_upsert_table(const dbsp_schema* t, const std::string& what) {
  std::string m = valid_schema(t, what, "table");
  if (!m.empty()) return m;
  if (t->n_key_lanes == 0) return what + ": table has no key lanes; a command replaces a key's row";
  const int L = t->n_key_lanes + t->n_val_lanes;
  if (L > DBSP_MAX_LANES - 1)
    return what + ": table has " + num(L) + " lanes; the command lane takes the 8th, so a table has at most 7";
  return "";
}
// upsert_commands: a valid table, and sequence numbers seq0 .. seq0 + n - 1 that fit 63 bits (the command word is
// the sequence number shifted left by one, the insert bit below it).
inline std::string valid_upsert(const dbsp_schema* table, uint64_t n, uint64_t seq0) {
  const std::string what = "upsert_commands";
  std::string m = valid_upsert_table(table, what);
  if (!m.empty()) return m;
  if (seq0 > (1ull << 63) || n > (1ull << 63) - seq0)
    return what + ": seq0 + n = " + num(seq0) + " + " + num(n) + " exceeds 2^63; a command's sequence number has 63 bits";
  return "";
}
// upsert_delta: a valid table, and a command batch with the schema upsert_commands gives for it.
inline std::string valid_upsert(const dbsp_schema& cmds, const dbsp_schema& table) {
  const std::string what = "upsert_delta";
  std::string m = valid_upsert_table(&table, what);
  if (!m.empty()) return m;
  if (!same_schema(cmds, upsert_command_schema(table)))
    return what + ": cmds must have the table's key lanes, then a u64 command lane and the table's value lanes";
  return "";
}

// ---- snapshot files (dbsp_spine_save / dbsp_spine_load)---------------------------------------------------------
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
