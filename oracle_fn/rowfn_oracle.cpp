// rowfn_oracle.cpp — the CPU oracle with row functions (dbsp_rowfn, include/dbsp_b200.h): the whole oracle of
// oracle/dbsp_oracle.cpp, unchanged, plus the `_fn` and `_fanout` entry points, dbsp_antijoin_delta,
// dbsp_aggregate_fold, the set / map input calls (dbsp_upsert_commands, dbsp_upsert_delta) and dbsp_rolling_aggregate, in one translation unit
// so that they build on its batches, traces, consolidation and error text.  The oracle's own library stays the checker
// of every `dbsp_proj` test; this one (libdbsp_oracle_fn.so, test infrastructure like it, never linked into the
// product) is the checker of the row-function, antijoin, fold, upsert and rolling aggregate tests.  The interpreter below is written apart from the CUDA library's; validate.h is shared,
// so both libraries refuse the same programs with the same texts.
#include <deque>

#include "../oracle/dbsp_oracle.cpp"

namespace {

// The postfix program over a stack; afterwards st[0..L) are the output lanes and st[L] the keep flag.  The arithmetic
// follows Rust's wrapping_* integer methods with x / 0 = x % 0 = 0 (DESIGN §2).  j: the output a fan-out generates,
// pushed by DBSP_SRC_FANOUT; acc / w: a fold's accumulator and the value's weight, pushed by DBSP_SRC_ACC /
// DBSP_SRC_WEIGHT (each validated away in the calls that do not have it).
void run_rowfn(const dbsp_rowfn& f, const Env& e, u64* st, u64 j = 0, const u64* acc = nullptr, i64 w = 0) {
  int sp = 0;
  for (int pc = 0; pc < f.n_insn; pc++) {
    const dbsp_insn& in = f.code[pc];
    if (in.op == DBSP_FN_PUSH) {
      dbsp_src s;
      s.kind = in.kind;
      s.idx = in.idx;
      s.cst = in.cst;
      st[sp++] = in.kind == DBSP_SRC_FANOUT ? j : in.kind == DBSP_SRC_ACC ? acc[in.idx] : in.kind == DBSP_SRC_WEIGHT ? (u64)w
                                                                                                         : src_val(s, e);
      continue;
    }
    const int pops = dbsp_validate::rowfn_arity(in.op);
    const u64 a = st[sp - pops], b = pops >= 2 ? st[sp - pops + 1] : 0, c = pops == 3 ? st[sp - 1] : 0;
    const i64 sa = (i64)a, sb = (i64)b;
    u64 r = 0;
    switch (in.op) {
      case DBSP_FN_NEG: r = (u64)0 - a; break;
      case DBSP_FN_ABS: r = sa < 0 ? (u64)0 - a : a; break;
      case DBSP_FN_BNOT: r = ~a; break;
      case DBSP_FN_LNOT: r = a == 0; break;
      case DBSP_FN_ADD: r = a + b; break;
      case DBSP_FN_SUB: r = a - b; break;
      case DBSP_FN_MUL: r = a * b; break;
      case DBSP_FN_DIV: r = sb == 0 ? 0 : sb == -1 ? (u64)0 - a : (u64)(sa / sb); break;   // MIN / -1 would trap
      case DBSP_FN_REM: r = (sb == 0 || sb == -1) ? 0 : (u64)(sa % sb); break;
      case DBSP_FN_DIVU: r = b == 0 ? 0 : a / b; break;
      case DBSP_FN_REMU: r = b == 0 ? 0 : a % b; break;
      case DBSP_FN_MIN: r = (u64)std::min(sa, sb); break;
      case DBSP_FN_MAX: r = (u64)std::max(sa, sb); break;
      case DBSP_FN_MINU: r = std::min(a, b); break;
      case DBSP_FN_MAXU: r = std::max(a, b); break;
      case DBSP_FN_AND: r = a & b; break;
      case DBSP_FN_OR: r = a | b; break;
      case DBSP_FN_XOR: r = a ^ b; break;
      case DBSP_FN_SHL: r = a << (b % 64); break;
      case DBSP_FN_SHR: r = a >> (b % 64); break;
      case DBSP_FN_SAR: r = (u64)(sa >> (b % 64)); break;
      case DBSP_FN_EQ: r = a == b; break;
      case DBSP_FN_NE: r = a != b; break;
      case DBSP_FN_LT: r = sa < sb; break;
      case DBSP_FN_LE: r = sa <= sb; break;
      case DBSP_FN_GT: r = sa > sb; break;
      case DBSP_FN_GE: r = sa >= sb; break;
      case DBSP_FN_LTU: r = a < b; break;
      case DBSP_FN_LEU: r = a <= b; break;
      case DBSP_FN_GTU: r = a > b; break;
      case DBSP_FN_GEU: r = a >= b; break;
      case DBSP_FN_IN: r = a < 64 && ((b >> a) & 1); break;
      case DBSP_FN_SELECT: r = a != 0 ? b : c; break;
    }
    sp -= pops;
    st[sp++] = r;
  }
}
// the output row and whether the program keeps it
bool project_fn(const dbsp_rowfn& f, const Env& e, u64* row, u64 j = 0) {
  u64 st[DBSP_MAX_STACK];
  run_rowfn(f, e, st, j);
  const int nl = f.out_schema.n_key_lanes + f.out_schema.n_val_lanes;
  for (int l = 0; l < nl; l++) row[l] = st[l];
  return st[nl] != 0;
}

// Join::eval (operator/join.rs:436-473) with a row function as join_func: the merge walk of join_into.
void join_into_fn(const Batch& L, const Batch& R, const dbsp_rowfn& f, bool swap, Tuples& out) {
  size_t i = 0, j = 0;
  u64 key[MAXL], v1[MAXL], v2[MAXL], row[MAXL];
  while (i < L.K.n && j < R.K.n) {
    int c = cmp_rows(L.K, i, R.K, j);
    if (c < 0) { i = i + advance(i, L.K.n, [&](size_t x) { return cmp_rows(L.K, x, R.K, j) < 0; }); }
    else if (c > 0) { j = j + advance(j, R.K.n, [&](size_t x) { return cmp_rows(R.K, x, L.K, i) < 0; }); }
    else {
      L.K.get(i, key);
      size_t l0, l1, r0, r1;
      L.vrange(i, l0, l1);
      R.vrange(j, r0, r1);
      for (size_t a = l0; a < l1; a++) {
        if (L.indexed()) L.V.get(a, v1);
        for (size_t b = r0; b < r1; b++) {
          if (R.indexed()) R.V.get(b, v2);
          Env e = swap ? Env{key, v2, v1} : Env{key, v1, v2};
          if (project_fn(f, e, row)) out.push(row, (i64)((u64)L.w[a] * (u64)R.w[b]));
        }
      }
      i++; j++;
    }
  }
}

// n_out == 0: a plain row function (`_fn`); otherwise a fan-out whose program runs for j = 0 .. n_out-1 per row.
int32_t table_to_batch_fn(const u64* const* cols, uint32_t ncols, const i64* w, u64 n, const dbsp_rowfn* fn, orc_batch** out,
                          uint32_t n_out = 0) {
  const unsigned used = dv::rowfn_table_mask(*fn);
  Tuples t(fn->out_schema);
  u64 lv[MAXL] = {0}, row[MAXL];
  for (u64 i = 0; i < n; i++) {
    for (uint32_t c = 0; c < ncols; c++) if ((used >> c) & 1) lv[c] = cols[c][i];
    Env e{lv, lv, lv};
    for (u64 j = 0; j < std::max<u64>(n_out, 1); j++)
      if (project_fn(*fn, e, row, j)) t.push(row, w ? w[i] : 1);
  }
  *out = wrap(t.build());
  return DBSP_OK;
}

// Upsert::eval for one key (operator/upsert.rs:161-208): retract the key's current values in the output trace, insert
// the new one (if any), and push what does not cancel.
void upsert_key(Builder& bld, const Spine& out_tr, const u64* key, const u64* newv, bool has_new) {
  const dbsp_schema& os = out_tr.s;
  const int nov = os.n_val_lanes;
  std::vector<std::pair<KV, i64>> grp;
  key_group(out_tr, key, grp);
  std::vector<std::pair<std::vector<u64>, i64>> upd;
  if (has_new) upd.push_back({std::vector<u64>(newv, newv + nov), 1});
  for (auto& g : grp)
    if (g.second != 0) {
      std::vector<u64> v(nov);
      g.first.b->V.get(g.first.pos, v.data());
      upd.push_back({v, (i64)((u64)0 - (u64)g.second)});
    }
  const uint8_t* vty = os.lane_types + os.n_key_lanes;
  std::sort(upd.begin(), upd.end(), [&](auto& a, auto& b) { return cmp_tuples(vty, nov, a.first.data(), b.first.data()) < 0; });
  for (size_t i = 0; i < upd.size();) {
    size_t j = i;
    i64 sum = 0;
    for (; j < upd.size() && cmp_tuples(vty, nov, upd[i].first.data(), upd[j].first.data()) == 0; j++)
      sum = (i64)((u64)sum + (u64)upd[j].second);
    if (sum != 0) bld.push(key, upd[i].first.data(), sum);
    i = j;
  }
}

// range.rs's timestamp arithmetic in the TS lane's type (i64 when sgn), in 128-bit integers: checked forms return
// false when the result leaves the type, saturating ones clamp to it.
struct RollTs {
  bool sgn;
  __int128 lo() const { return sgn ? (__int128)INT64_MIN : 0; }
  __int128 hi() const { return sgn ? (__int128)INT64_MAX : (__int128)~0ull; }
  __int128 val(u64 x) const { return sgn ? (__int128)(i64)x : (__int128)x; }
  bool fits(__int128 v) const { return v >= lo() && v <= hi(); }
  u64 clamp(__int128 v) const { return (u64)(v < lo() ? lo() : v > hi() ? hi() : v); }
  bool lt(u64 a, u64 b) const { return val(a) < val(b); }
  // RelRange::range_of / affected_range_of
  bool range_of(const dbsp_rel_range& r, u64 ts, u64* from, u64* to) const {
    const __int128 t = val(ts);
    const __int128 f = r.from_after ? t + r.from_off : t - r.from_off, e = r.to_after ? t + r.to_off : t - r.to_off;
    if ((r.from_after && !fits(f)) || (!r.to_after && !fits(e))) return false;
    *from = clamp(f);
    *to = clamp(e);
    return true;
  }
  bool affected_of(const dbsp_rel_range& r, u64 ts, u64* from, u64* to) const {
    const __int128 t = val(ts);
    const __int128 f = r.to_after ? t - r.to_off : t + r.to_off, e = r.from_after ? t - r.from_off : t + r.from_off;
    if ((!r.to_after && !fits(f)) || (r.from_after && !fits(e))) return false;
    *from = clamp(f);
    *to = clamp(e);
    return true;
  }
};

}  // namespace

extern "C" {

// PartitionedRollingAggregate::eval (operator/time_series/rolling_aggregate.rs:436-604) as it reads, with the radix
// tree replaced by a walk of each affected partition in ts order: per partition key of delta, the affected ranges
// (affected_range_of(d) and [d, d] per delta time, merged), out_trace's rows in them retracted, then the partition's
// rows of in_trace (weights summed over the batches, zeros skipped) walked once with two window ends that only move
// forward: running sums for LINEAR, a monotone deque of candidates for MAX / MIN.  Written apart from the CUDA
// library's gather, prefix sums and sparse table.
int32_t orc_rolling_aggregate(orc_ctx* c, const orc_batch* delta, const orc_spine* in_tr, const orc_spine* out_tr,
                              const dbsp_rel_range* range, int32_t kind, const dbsp_rowfn* f, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::valid_rolling(out, S(delta), S(in_tr), S(out_tr), range, kind, f));
  const Batch& D = *delta->p;
  const dbsp_schema& os = out_tr->s.s;
  const int nk = D.s.n_key_lanes, nvv = D.s.n_val_lanes - 1, n_agg = os.n_val_lanes - 2;
  const RollTs T{D.s.lane_types[nk] == DBSP_I64};
  const uint8_t* vty = D.s.lane_types + nk + 1;
  Tuples t(os);
  std::vector<std::pair<KV, i64>> grp;
  u64 row[MAXL], v[MAXL] = {0}, st[DBSP_MAX_STACK];
  for (size_t k = 0; k < D.K.n; k++) {
    D.K.get(k, row);
    // affected ranges, sorted and merged
    std::vector<std::pair<u64, u64>> iv;
    size_t lo, hi;
    D.vrange(k, lo, hi);
    for (size_t j = lo; j < hi; j++) {
      const u64 d = D.V.c[0][j];
      u64 a, b;
      iv.push_back({d, d});
      if (T.affected_of(*range, d, &a, &b)) iv.push_back({a, b});
    }
    std::sort(iv.begin(), iv.end(), [&](auto& x, auto& y) { return T.lt(x.first, y.first); });
    std::vector<std::pair<u64, u64>> ranges;
    for (auto& r : iv) {
      if (!ranges.empty() && !T.lt(ranges.back().second, r.first)) {
        if (T.lt(ranges.back().second, r.second)) ranges.back().second = r.second;
      } else {
        ranges.push_back(r);
      }
    }
    auto affected = [&](size_t& ri, u64 ts) {   // ts ascending across calls
      while (ri < ranges.size() && T.lt(ranges[ri].second, ts)) ri++;
      return ri < ranges.size() && !T.lt(ts, ranges[ri].first);
    };
    // retract the old outputs
    key_group(out_tr->s, row, grp);
    size_t ri = 0;
    for (auto& g : grp) {
      if (g.second == 0) continue;
      g.first.b->V.get(g.first.pos, row + nk);
      if (affected(ri, row[nk])) t.push(row, (i64)((u64)0 - (u64)g.second));
    }
    // the partition's rows in (ts, v) order
    key_group(in_tr->s, row, grp);
    std::vector<u64> ts;
    std::vector<i64> w;
    std::vector<std::vector<u64>> vals;
    for (auto& g : grp) {
      if (g.second == 0) continue;
      g.first.b->V.get(g.first.pos, v);
      ts.push_back(v[0]);
      w.push_back(g.second);
      vals.emplace_back(v + 1, v + 1 + nvv);
    }
    const size_t n = ts.size();
    // LINEAR: each row's term f(pk, v) * w; MAX / MIN: rows compared by V
    std::vector<std::vector<u64>> term(n, std::vector<u64>(std::max(n_agg, 0), 0));
    if (kind == DBSP_ROLLING_LINEAR)
      for (size_t j = 0; j < n; j++) {
        run_rowfn(*f, Env{row, vals[j].data(), vals[j].data()}, st);
        if (st[n_agg] != 0)
          for (int l = 0; l < n_agg; l++) term[j][l] = st[l] * (u64)w[j];
      }
    const int sign = kind == DBSP_ROLLING_MAX ? 1 : -1;
    auto not_worse = [&](size_t a, size_t b) {   // row a's V at least as good as row b's
      return sign * cmp_tuples(vty, nvv, vals[a].data(), vals[b].data()) >= 0;
    };
    std::vector<u64> sum(std::max(n_agg, 0), 0);
    std::deque<size_t> dq;
    size_t wl = 0, wh = 0;   // the window is rows [wl, wh)
    ri = 0;
    for (size_t j = 0; j < n;) {
      size_t e = j;
      bool pos = false;
      for (; e < n && ts[e] == ts[j]; e++) pos = pos || w[e] > 0;
      u64 from, to;
      if (pos && affected(ri, ts[j]) && T.range_of(*range, ts[j], &from, &to)) {
        for (; wh < n && !T.lt(to, ts[wh]); wh++) {
          for (int l = 0; l < n_agg; l++) sum[l] += term[wh][l];
          if (kind != DBSP_ROLLING_LINEAR) {
            while (!dq.empty() && not_worse(wh, dq.back())) dq.pop_back();
            dq.push_back(wh);
          }
        }
        for (; wl < wh && T.lt(ts[wl], from); wl++)
          for (int l = 0; l < n_agg; l++) sum[l] -= term[wl][l];
        while (!dq.empty() && dq.front() < wl) dq.pop_front();
        row[nk] = ts[j];
        row[nk + 1] = wl < wh ? 1 : 0;
        for (int l = 0; l < n_agg; l++)
          row[nk + 2 + l] = wl >= wh ? 0 : kind == DBSP_ROLLING_LINEAR ? sum[l] : vals[dq.front()][l];
        t.push(row, 1);
      }
      j = e;
    }
  }
  *out = wrap(t.build());
  return DBSP_OK;
}

int32_t orc_batch_from_table_fn(orc_ctx* c, const u64* const* cols, uint32_t ncols, const i64* w, u64 n, int32_t,
                                const dbsp_rowfn* fn, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_table(WHAT, out, cols, ncols, n, fn));
  return table_to_batch_fn(cols, ncols, w, n, fn, out);
}

int32_t orc_batch_from_upload_fn(orc_ctx* c, orc_upload* u, const dbsp_rowfn* fn, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_upload(WHAT, out, upload_of(u, c), fn));
  return table_to_batch_fn(u->cols, u->n_cols, u->w, u->n, fn, out);
}

uint32_t orc_rowfn_table_mask(const dbsp_rowfn* fn) { return dv::checked_table_mask(fn, WHAT); }

// flat_map_index over a raw table with a fan-out (filter_map.rs:124-160: the closure returns an iterator).
int32_t orc_batch_from_table_fanout(orc_ctx* c, const u64* const* cols, uint32_t ncols, const i64* w, u64 n, int32_t,
                                    const dbsp_rowfn* fn, uint32_t n_out, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_table(WHAT, out, cols, ncols, n, fn, n_out));
  return table_to_batch_fn(cols, ncols, w, n, fn, out, n_out);
}

int32_t orc_batch_from_upload_fanout(orc_ctx* c, orc_upload* u, const dbsp_rowfn* fn, uint32_t n_out, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_upload(WHAT, out, upload_of(u, c), fn, n_out));
  return table_to_batch_fn(u->cols, u->n_cols, u->w, u->n, fn, out, n_out);
}

// antijoin (operator/join.rs:294-320) incrementally, as the formula reads: a delta row (k, v1, w) with N(k) distinct
// values on the other side gets w·(1 − N(k)), and every trace row (k, v1, w') of a key whose count changed by dN
// adds −dN·w'.  Written apart from the CUDA library's lookups and gather.
int32_t orc_antijoin_delta(orc_ctx* c, const orc_batch* delta, const orc_spine* tr, const orc_batch* kd,
                           const orc_spine* kt, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::valid_antijoin(out, S(delta), S(tr), S(kd), S(kt)));
  const Batch& D = *delta->p;
  const int nk = D.s.n_key_lanes;
  Tuples t(D.s);
  std::vector<std::pair<KV, i64>> grp;
  u64 row[MAXL];
  for (size_t k = 0; k < D.K.n; k++) {
    D.K.get(k, row);
    key_group(kt->s, row, grp);   // no value lanes: one group, the key's count summed over the batches
    const u64 one_minus_n = (u64)1 - (u64)(grp.empty() ? 0 : grp[0].second);
    size_t lo, hi;
    D.vrange(k, lo, hi);
    for (size_t v = lo; v < hi; v++) {
      if (D.indexed()) D.V.get(v, row + nk);
      t.push(row, (i64)((u64)D.w[v] * one_minus_n));
    }
  }
  const Batch& KD = *kd->p;
  for (size_t k = 0; k < KD.K.n; k++) {
    KD.K.get(k, row);
    for (auto& bp : tr->s.batches) {
      const Batch& b = *bp;
      const size_t i = seek_key(b, 0, row);
      if (i >= b.K.n || cmp_row_tuple(b.K, i, row) != 0) continue;
      size_t lo, hi;
      b.vrange(i, lo, hi);
      for (size_t v = lo; v < hi; v++) {
        if (b.indexed()) b.V.get(v, row + nk);
        t.push(row, (i64)((u64)0 - (u64)KD.w[k] * (u64)b.w[v]));
      }
    }
  }
  *out = wrap(t.build());
  return DBSP_OK;
}

// AggregateIncremental + Upsert with a Fold, as fold.rs:60-75 reads: per key of delta, the key's values in value
// order with their weights summed over the batches; a value of weight 0 is skipped, every other one runs `step`
// (whose keep flag decides whether its words become the accumulator); a non-empty key's output row is output(acc)
// unless the output program drops it.  Written apart from the CUDA library's gather and per-key walk.
int32_t orc_aggregate_fold(orc_ctx* c, const orc_batch* delta, const orc_spine* in_tr, const orc_spine* out_tr,
                           const dbsp_fold* fold, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::valid_fold(out, S(delta), S(in_tr), S(out_tr), fold));
  const Batch& D = *delta->p;
  const int n_acc = fold->n_acc, nov = out_tr->s.s.n_val_lanes;
  const dbsp_rowfn step = dv::fold_step_rowfn(*fold);
  Builder bld(out_tr->s.s);
  std::vector<std::pair<KV, i64>> grp;
  u64 key[MAXL], val[MAXL] = {0}, acc[DBSP_MAX_ACC], st[DBSP_MAX_STACK];
  for (size_t k = 0; k < D.K.n; k++) {
    D.K.get(k, key);
    key_group(in_tr->s, key, grp);
    std::copy(fold->init, fold->init + n_acc, acc);
    bool non_empty = false;
    for (auto& g : grp) {
      if (g.second == 0) continue;
      non_empty = true;
      if (g.first.b->indexed()) g.first.b->V.get(g.first.pos, val);
      run_rowfn(step, Env{key, val, val}, st, 0, acc, g.second);
      if (st[n_acc] != 0) std::copy(st, st + n_acc, acc);
    }
    bool has_new = false;
    if (non_empty) {
      run_rowfn(fold->output, Env{key, val, val}, st, 0, acc, 0);
      has_new = st[nov] != 0;
    }
    upsert_key(bld, out_tr->s, key, st, has_new);
  }
  *out = wrap(bld.done());
  return DBSP_OK;
}

// The commands of a set / map input as a batch: (key, command word, value) rows, a delete's values 0, consolidated.
int32_t orc_upsert_commands(orc_ctx* c, const dbsp_schema* table, const u64* const* cols, const uint8_t* insert, u64 n,
                            u64 seq0, int32_t, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::valid_upsert(out, table, cols, n, seq0));
  const int nk = table->n_key_lanes, nv = table->n_val_lanes;
  Tuples t(dv::upsert_command_schema(*table));
  u64 row[MAXL];
  for (u64 i = 0; i < n; i++) {
    const bool ins = insert == nullptr || insert[i] != 0;
    for (int l = 0; l < nk; l++) row[l] = cols[l][i];
    row[nk] = ((seq0 + i) << 1) | (ins ? 1 : 0);
    for (int l = 0; l < nv; l++) row[nk + 1 + l] = ins ? cols[nk + l][i] : 0;
    t.push(row, 1);
  }
  *out = wrap(t.build());
  return DBSP_OK;
}

// add_upsert (operator/input.rs:141-160) and Upsert::eval (operator/upsert.rs:161-208), as they read: the commands in
// sequence order, stable-sorted by key, the last command of each key kept, then per key a seek into the table's trace
// that retracts its current values and inserts the new one.  Written apart from the CUDA library's flags and
// compactions.
int32_t orc_upsert_delta(orc_ctx* c, const orc_batch* cmds, const orc_spine* table, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::valid_upsert(out, S(cmds), S(table)));
  const Batch& C = *cmds->p;
  const dbsp_schema& ts = table->s.s;
  // the commands: row j of the batch, its key at kof[j], its command word in value lane 0, its values after it
  std::vector<uint32_t> kof(C.len());
  for (size_t k = 0; k < C.K.n; k++)
    for (size_t j = C.offs[k]; j < C.offs[k + 1]; j++) kof[j] = (uint32_t)k;
  const std::vector<u64>& word = C.V.c[0];
  std::vector<size_t> v(C.len());
  for (size_t j = 0; j < v.size(); j++) v[j] = j;
  std::sort(v.begin(), v.end(), [&](size_t a, size_t b) { return word[a] < word[b]; });   // arrival order
  std::stable_sort(v.begin(), v.end(), [&](size_t a, size_t b) { return cmp_rows(C.K, kof[a], C.K, kof[b]) < 0; });
  Builder bld(ts);
  u64 key[MAXL], cv[MAXL];
  for (size_t i = 0; i < v.size(); i++) {
    if (i + 1 < v.size() && kof[v[i]] == kof[v[i + 1]]) continue;   // a later command of the key follows
    C.K.get(kof[v[i]], key);
    C.V.get(v[i], cv);
    upsert_key(bld, table->s, key, cv + 1, (cv[0] & 1) != 0);
  }
  *out = wrap(bld.done());
  return DBSP_OK;
}

uint32_t orc_fanout_table_mask(const dbsp_rowfn* fn) { return dv::checked_table_mask(fn, WHAT, dv::SRC_BIT_FANOUT); }

// JoinTrace::eval with Time = () (operator/join.rs:732-863): delta joined with every batch of the trace.
int32_t orc_join_delta_trace_fn(orc_ctx* c, const orc_batch* delta, const orc_spine* tr, const dbsp_rowfn* fn,
                                int32_t delta_is_left, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_join(WHAT, out, S(delta), S(tr), delta_is_left, fn));
  Tuples t(fn->out_schema);
  for (auto& b : tr->s.batches) join_into_fn(*delta->p, *b, *fn, !delta_is_left, t);
  *out = wrap(t.build());
  return DBSP_OK;
}

int32_t orc_join_batches_fn(orc_ctx* c, const orc_batch* l, const orc_batch* r, const dbsp_rowfn* fn, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_join(WHAT, out, S(l), S(r), fn));
  Tuples t(fn->out_schema);
  join_into_fn(*l->p, *r->p, *fn, false, t);
  *out = wrap(t.build());
  return DBSP_OK;
}

// weigh (operator/aggregate/mod.rs:297-323) with a one-lane row function: a row the program drops adds nothing to
// the sum, nor (WEIGH_AVG) to the count.
int32_t orc_weigh_fn(orc_ctx* c, const orc_batch* b, const dbsp_rowfn* f, int32_t mode, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_weigh(out, S(b), f, mode));
  const Batch& B = *b->p;
  dbsp_schema s = B.s;
  s.n_val_lanes = 0;
  if (mode == DBSP_WEIGH_AVG) { s.lane_types[s.n_key_lanes] = DBSP_U64; s.n_key_lanes++; }
  Builder bld(s);
  u64 key[MAXL], val[MAXL] = {0}, fv;
  for (size_t k = 0; k < B.K.n; k++) {
    B.K.get(k, key);
    size_t lo, hi;
    B.vrange(k, lo, hi);
    i64 agg = 0, cnt = 0;
    for (size_t v = lo; v < hi; v++) {
      if (B.indexed()) B.V.get(v, val);
      Env e{key, val, val};
      if (!project_fn(*f, e, &fv)) continue;
      agg = (i64)((u64)agg + fv * (u64)B.w[v]);
      cnt = (i64)((u64)cnt + (u64)B.w[v]);
    }
    if (mode == DBSP_WEIGH_AVG) {
      key[B.s.n_key_lanes] = 0; if (agg != 0) bld.push(key, nullptr, agg);
      key[B.s.n_key_lanes] = 1; if (cnt != 0) bld.push(key, nullptr, cnt);
    } else if (agg != 0) {
      bld.push(key, nullptr, agg);
    }
  }
  *out = wrap(bld.done());
  return DBSP_OK;
}

// Map/FlatMap/Index::eval + from_tuples (operator/filter_map.rs:563-577,700-724); n_out == 0: no fan-out.
static int32_t map_index_fn(const orc_batch* b, const dbsp_rowfn* fn, uint32_t n_out, orc_batch** out) {
  const Batch& B = *b->p;
  Tuples t(fn->out_schema);
  u64 key[MAXL], val[MAXL] = {0}, row[MAXL];
  for (size_t k = 0; k < B.K.n; k++) {
    B.K.get(k, key);
    size_t lo, hi;
    B.vrange(k, lo, hi);
    for (size_t v = lo; v < hi; v++) {
      if (B.indexed()) B.V.get(v, val);
      Env e{key, val, val};
      for (u64 j = 0; j < std::max<u64>(n_out, 1); j++)
        if (project_fn(*fn, e, row, j)) t.push(row, B.w[v]);
    }
  }
  *out = wrap(t.build());
  return DBSP_OK;
}

int32_t orc_map_index_fn(orc_ctx* c, const orc_batch* b, const dbsp_rowfn* fn, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_map_index(WHAT, out, S(b), fn));
  return map_index_fn(b, fn, 0, out);
}

// flat_map / flat_map_index of a batch with a fan-out: j = 0 .. n_out-1 per row, in one pass.
int32_t orc_map_index_fanout(orc_ctx* c, const orc_batch* b, const dbsp_rowfn* fn, uint32_t n_out, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_map_index(WHAT, out, S(b), b ? b->p->len() : 0, fn, n_out));
  return map_index_fn(b, fn, n_out, out);
}

}  // extern "C"
