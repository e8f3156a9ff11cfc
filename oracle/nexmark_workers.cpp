// nexmark_workers.cpp — the CPU arm of bench.py: N replicas of a Nexmark query circuit on N host threads.
//
// TEST / BASELINE INFRASTRUCTURE (lives under oracle/, links libdbsp_oracle.so): used only by bench.py's
// `cpu_baseline` / `--impl reference` legs and by tests/test_oracle_workers.py.  Never loaded by the product.
//
// Execution model = the reference's: `Runtime::run` spawns one worker thread per circuit replica
// (crates/dbsp/src/circuit/runtime.rs:137-180); every keyed operator is preceded by `shard()`
// (operator/communication/shard.rs:106-162), whose all-to-all goes through shared in-process mailboxes
// with one round per exchange (operator/communication/exchange.rs:45-64,128-200).  The circuits are the
// queries of crates/nexmark/src/queries/{q3,q4,q7}.rs restated over the oracle's operator entry points
// (the same sequence of operator calls dbsp_b200/nexmark/queries.py + circuit.py make); there is no
// interpreter between steps — a step is one pass of every worker over its slice of the step's events.
#include <atomic>
#include <chrono>
#include <cstdint>
#include <cstring>
#include <thread>
#include <vector>

#include "../include/dbsp_b200.h"

typedef uint64_t u64;
typedef int64_t i64;

struct orc_ctx;
struct orc_batch;
struct orc_spine;
extern "C" {
int32_t orc_ctx_create(int32_t, orc_ctx**);
int32_t orc_ctx_destroy(orc_ctx*);
int32_t orc_batch_from_table(orc_ctx*, const u64* const*, uint32_t, const i64*, u64, int32_t, const dbsp_proj*, orc_batch**);
int32_t orc_batch_empty(orc_ctx*, const dbsp_schema*, orc_batch**);
int32_t orc_batch_merge(orc_ctx*, const orc_batch*, const orc_batch*, orc_batch**);
int32_t orc_batch_reindex(orc_ctx*, const orc_batch*, uint32_t, orc_batch**);
int32_t orc_batch_len(const orc_batch*, u64*);
int32_t orc_batch_key_count(orc_ctx*, const orc_batch*, u64*);
int32_t orc_batch_download_csr(orc_ctx*, const orc_batch*, u64* const*, u64*, u64* const*, i64*);
int32_t orc_batch_last_key(orc_ctx*, const orc_batch*, u64*, int32_t*);
int32_t orc_batch_free(orc_batch*);
int32_t orc_spine_new(orc_ctx*, const dbsp_schema*, orc_spine**);
int32_t orc_spine_insert(orc_ctx*, orc_spine*, const orc_batch*);
int32_t orc_spine_truncate_keys_below(orc_ctx*, orc_spine*, const u64*);
int32_t orc_spine_free(orc_spine*);
int32_t orc_join_delta_trace(orc_ctx*, const orc_batch*, const orc_spine*, const dbsp_proj*, int32_t, orc_batch**);
int32_t orc_aggregate_delta(orc_ctx*, const orc_batch*, const orc_spine*, const orc_spine*, int32_t, orc_batch**);
int32_t orc_weigh(orc_ctx*, const orc_batch*, const dbsp_expr*, int32_t, orc_batch**);
int32_t orc_window_delta(orc_ctx*, const orc_spine*, const orc_batch*, int32_t, const u64*, const u64*, const u64*, const u64*, orc_batch**);
int32_t orc_map_index(orc_ctx*, const orc_batch*, const dbsp_proj*, orc_batch**);
int32_t orc_shard_partition(orc_ctx*, const orc_batch*, uint32_t, orc_batch**);
}

namespace {

// ---- declarative closures (the Proj objects of nexmark/queries.py) --------------------------------
dbsp_schema schema(const char* key, const char* val) {
  dbsp_schema s;
  memset(&s, 0, sizeof(s));
  s.n_key_lanes = (uint8_t)strlen(key);
  s.n_val_lanes = (uint8_t)strlen(val);
  int i = 0;
  for (const char* p = key; *p; p++) s.lane_types[i++] = *p == 'i' ? DBSP_I64 : DBSP_U64;
  for (const char* p = val; *p; p++) s.lane_types[i++] = *p == 'i' ? DBSP_I64 : DBSP_U64;
  return s;
}
dbsp_src src(int kind, int idx, i64 cst = 0) {
  dbsp_src s;
  memset(&s, 0, sizeof(s));
  s.kind = (uint8_t)kind;
  s.idx = (uint8_t)idx;
  s.cst = cst;
  return s;
}
dbsp_src K(int i) { return src(DBSP_SRC_KEY, i); }
dbsp_src LV(int i) { return src(DBSP_SRC_LVAL, i); }
dbsp_src RV(int i) { return src(DBSP_SRC_RVAL, i); }
dbsp_src CST(i64 c) { return src(DBSP_SRC_CONST, 0, c); }
dbsp_expr ex(int op, dbsp_src a, dbsp_src b = src(DBSP_SRC_CONST, 0)) {
  dbsp_expr e;
  memset(&e, 0, sizeof(e));
  e.op = (uint8_t)op;
  e.a = a;
  e.b = b;
  return e;
}
dbsp_pred pr(int cmp, dbsp_src a, dbsp_src b) {
  dbsp_pred p;
  memset(&p, 0, sizeof(p));
  p.cmp = (uint8_t)cmp;
  p.a = a;
  p.b = b;
  return p;
}
dbsp_proj proj(dbsp_schema s, std::vector<dbsp_expr> out, std::vector<dbsp_pred> where = {}) {
  dbsp_proj p;
  memset(&p, 0, sizeof(p));
  p.out_schema = s;
  p.n_pred = (uint8_t)where.size();
  for (size_t i = 0; i < out.size(); i++) p.out[i] = out[i];
  for (size_t i = 0; i < where.size(); i++) p.pred[i] = where[i];
  return p;
}
dbsp_expr cp(dbsp_src a) { return ex(DBSP_OP_COPY, a); }

// ---- in-process exchange (exchange.rs:45-64): box[src][dst] + a barrier per round ---------------------
struct Barrier {
  std::atomic<int> count{0};
  std::atomic<int> sense{0};
  int n;
  explicit Barrier(int n_) : n(n_) {}
  void wait() {
    const int s = sense.load(std::memory_order_acquire);
    if (count.fetch_add(1, std::memory_order_acq_rel) == n - 1) {
      count.store(0, std::memory_order_relaxed);
      sense.store(s ^ 1, std::memory_order_release);
    } else {
      int spins = 0;
      while (sense.load(std::memory_order_acquire) == s)
        if (++spins > 2000) std::this_thread::yield();
    }
  }
};

struct Shared {
  int T;
  Barrier bar;
  std::vector<orc_batch*> box;   // [stream][src][dst], 2 streams per round
  std::vector<u64> scalars;
  explicit Shared(int t) : T(t), bar(t), box((size_t)2 * t * t, nullptr), scalars((size_t)t, 0) {}
  orc_batch*& at(int stream, int s, int d) { return box[((size_t)stream * T + s) * T + d]; }
};

struct Worker {
  Shared* sh;
  int rank, T;
  orc_ctx* ctx = nullptr;

  orc_batch* merge_all(std::vector<orc_batch*> v) {   // receiver side of shard(): balanced merge (shard.rs:136-144)
    while (v.size() > 1) {
      std::vector<orc_batch*> nx;
      size_t i = 0;
      for (; i + 1 < v.size(); i += 2) {
        orc_batch* m = nullptr;
        orc_batch_merge(ctx, v[i], v[i + 1], &m);
        orc_batch_free(v[i]);
        orc_batch_free(v[i + 1]);
        nx.push_back(m);
      }
      if (i < v.size()) nx.push_back(v[i]);
      v.swap(nx);
    }
    return v[0];
  }
  // shard() of up to two streams in one exchange round; consumes the inputs
  void shard_many(orc_batch** bs, int ns) {
    if (T == 1) return;
    std::vector<orc_batch*> parts((size_t)T);
    for (int i = 0; i < ns; i++) {
      orc_shard_partition(ctx, bs[i], (uint32_t)T, parts.data());
      for (int d = 0; d < T; d++) sh->at(i, rank, d) = parts[d];
      orc_batch_free(bs[i]);
    }
    sh->bar.wait();
    for (int i = 0; i < ns; i++) {
      std::vector<orc_batch*> got((size_t)T);
      for (int s = 0; s < T; s++) got[s] = sh->at(i, s, rank);
      bs[i] = merge_all(got);
    }
    sh->bar.wait();   // every mailbox drained before the next round overwrites it
  }
  orc_batch* shard(orc_batch* b) { shard_many(&b, 1); return b; }
  orc_batch* gather0(orc_batch* b, const dbsp_schema& s) {   // gather (gather.rs:41-103) to worker 0
    if (T == 1) return b;
    sh->at(0, rank, 0) = b;
    sh->bar.wait();
    orc_batch* out = nullptr;
    if (rank == 0) {
      std::vector<orc_batch*> got((size_t)T);
      for (int s = 0; s < T; s++) got[s] = sh->at(0, s, 0);
      out = merge_all(got);
    } else {
      orc_batch_empty(ctx, &s, &out);
    }
    sh->bar.wait();
    return out;
  }
  u64 allreduce_max(u64 x) {   // watermark exchange (watermark.rs:53-70)
    if (T == 1) return x;
    sh->scalars[(size_t)rank] = x;
    sh->bar.wait();
    u64 m = 0;
    for (int i = 0; i < T; i++) m = std::max(m, sh->scalars[(size_t)i]);
    sh->bar.wait();
    return m;
  }
};

struct Slice {   // this worker's rows of one table of one step
  const u64* cols[5];
  u64 n;
};

struct Query {
  virtual ~Query() {}
  virtual orc_batch* step(Worker& w, const Slice& person, const Slice& auction, const Slice& bid) = 0;
  virtual dbsp_schema out_schema() const = 0;
};

orc_spine* new_spine(Worker& w, const dbsp_schema& s) {
  orc_spine* sp = nullptr;
  orc_spine_new(w.ctx, &s, &sp);
  return sp;
}
orc_batch* from_table(Worker& w, const Slice& t, const dbsp_proj& p) {
  orc_batch* b = nullptr;
  orc_batch_from_table(w.ctx, t.cols, 5, nullptr, t.n, 0, &p, &b);
  return b;
}
// join (operator/join.rs:180-292): delta_L |x| trace(R) + delta_R |x| z^-1 trace(L); consumes dl, dr
orc_batch* join_step(Worker& w, orc_batch* dl, orc_batch* dr, orc_spine* lt, orc_spine* rt, const dbsp_proj& pj) {
  orc_spine_insert(w.ctx, rt, dr);
  orc_batch *o1 = nullptr, *o2 = nullptr, *out = nullptr;
  orc_join_delta_trace(w.ctx, dl, rt, &pj, 1, &o1);
  orc_join_delta_trace(w.ctx, dr, lt, &pj, 0, &o2);
  orc_spine_insert(w.ctx, lt, dl);
  orc_batch_merge(w.ctx, o1, o2, &out);
  orc_batch_free(o1);
  orc_batch_free(o2);
  orc_batch_free(dl);
  orc_batch_free(dr);
  return out;
}
// aggregate (aggregate/mod.rs:204-244) + upsert: consumes d
orc_batch* aggregate_step(Worker& w, orc_batch* d, orc_spine* in_tr, orc_spine* out_tr, int kind) {
  orc_spine_insert(w.ctx, in_tr, d);
  orc_batch* out = nullptr;
  orc_aggregate_delta(w.ctx, d, in_tr, out_tr, kind, &out);
  orc_spine_insert(w.ctx, out_tr, out);
  orc_batch_free(d);
  return out;
}
orc_batch* map_index(Worker& w, orc_batch* b, const dbsp_proj& p, bool consume = true) {
  orc_batch* o = nullptr;
  orc_map_index(w.ctx, b, &p, &o);
  if (consume) orc_batch_free(b);
  return o;
}
orc_batch* reindex(Worker& w, orc_batch* b, uint32_t nk) {
  orc_batch* o = nullptr;
  orc_batch_reindex(w.ctx, b, nk, &o);
  orc_batch_free(b);
  return o;
}

// queries/q3.rs:35-63
struct Q3 : Query {
  dbsp_proj pa, pp, pj;
  orc_spine *lt, *rt;
  explicit Q3(Worker& w) {
    pa = proj(schema("u", "u"), {cp(LV(1)), cp(LV(0))}, {pr(DBSP_CMP_EQ, LV(2), CST(10))});
    pp = proj(schema("u", "uuu"), {cp(LV(0)), cp(LV(1)), cp(LV(2)), cp(LV(3))}, {pr(DBSP_CMP_IN, LV(3), CST((1 << 1) | (1 << 2) | (1 << 3)))});
    pj = proj(schema("uuuu", ""), {cp(RV(0)), cp(RV(1)), cp(RV(2)), cp(LV(0))});
    lt = new_spine(w, pa.out_schema);
    rt = new_spine(w, pp.out_schema);
  }
  dbsp_schema out_schema() const override { return pj.out_schema; }
  orc_batch* step(Worker& w, const Slice& person, const Slice& auction, const Slice&) override {
    orc_batch* bs[2] = {from_table(w, auction, pa), from_table(w, person, pp)};
    w.shard_many(bs, 2);
    return join_step(w, bs[0], bs[1], lt, rt, pj);
  }
};

// queries/q4.rs:43-83
struct Q4 : Query {
  dbsp_proj pa, pb, pj, pcat, pavg, pfin;
  dbsp_expr fw;
  orc_spine *lt, *rt, *max_in, *max_out, *avg_in, *avg_out;
  explicit Q4(Worker& w) {
    pa = proj(schema("u", "uuu"), {cp(LV(0)), cp(LV(2)), cp(LV(3)), cp(LV(4))});
    pb = proj(schema("u", "uu"), {cp(LV(0)), cp(LV(2)), cp(LV(3))});
    pj = proj(schema("uu", "u"), {cp(K(0)), cp(LV(0)), cp(RV(0))}, {pr(DBSP_CMP_GE, RV(1), LV(1)), pr(DBSP_CMP_LE, RV(1), LV(2))});
    pcat = proj(schema("u", "u"), {cp(K(1)), cp(LV(0))});
    fw = cp(LV(0));
    // a key whose count sums to 0 has no average (as Stream.average)
    pavg = proj(schema("u", "i"), {cp(K(0)), ex(DBSP_OP_DIV, LV(0), LV(1))}, {pr(DBSP_CMP_NE, LV(1), CST(0))});
    pfin = proj(schema("uu", ""), {cp(K(0)), cp(LV(0))});
    lt = new_spine(w, pa.out_schema);
    rt = new_spine(w, pb.out_schema);
    max_in = new_spine(w, pj.out_schema);
    max_out = new_spine(w, pj.out_schema);
    avg_in = new_spine(w, schema("uu", ""));
    avg_out = new_spine(w, schema("u", "ii"));
  }
  dbsp_schema out_schema() const override { return pfin.out_schema; }
  orc_batch* step(Worker& w, const Slice&, const Slice& auction, const Slice& bid) override {
    orc_batch* bs[2] = {from_table(w, auction, pa), from_table(w, bid, pb)};
    w.shard_many(bs, 2);
    orc_batch* bfa = join_step(w, bs[0], bs[1], lt, rt, pj);            // bids_for_auctions
    orc_batch* win = aggregate_step(w, w.shard(bfa), max_in, max_out, DBSP_AGG_MAX);   // winning_bids
    orc_batch* bycat = map_index(w, win, pcat);
    orc_batch* wg = nullptr;                                            // average (average.rs:227-307)
    orc_weigh(w.ctx, bycat, &fw, DBSP_WEIGH_AVG, &wg);
    orc_batch_free(bycat);
    wg = reindex(w, w.shard(reindex(w, wg, 1)), 2);
    orc_batch* pair = aggregate_step(w, wg, avg_in, avg_out, DBSP_AGG_WCOUNT2);
    return map_index(w, map_index(w, pair, pavg), pfin);
  }
};

// queries/q7.rs:45-94
struct Q7 : Query {
  dbsp_proj pt, pprice, pneg, pmax, pj;
  orc_spine *wtrace, *loc_in, *loc_out, *min_in, *min_out, *lt, *rt;
  u64 wm = 0;
  bool has_prev = false;
  u64 prev_lo = 0, prev_hi = 0;
  explicit Q7(Worker& w) {
    pt = proj(schema("u", "uuuu"), {cp(LV(3)), cp(LV(0)), cp(LV(1)), cp(LV(2)), cp(LV(4))});
    pprice = proj(schema("u", "uuuuu"), {cp(LV(2)), cp(LV(0)), cp(LV(1)), cp(LV(2)), cp(K(0)), cp(LV(3))});
    pneg = proj(schema("", "i"), {ex(DBSP_OP_NEG, LV(2))});
    pmax = proj(schema("u", ""), {ex(DBSP_OP_NEG, LV(0))});
    pj = proj(schema("uuuuu", ""), {cp(RV(0)), cp(RV(1)), cp(RV(2)), cp(RV(3)), cp(RV(4))});
    wtrace = new_spine(w, pt.out_schema);
    loc_in = new_spine(w, pneg.out_schema);
    loc_out = new_spine(w, pneg.out_schema);
    min_in = new_spine(w, pneg.out_schema);
    min_out = new_spine(w, pneg.out_schema);
    lt = new_spine(w, pmax.out_schema);
    rt = new_spine(w, pprice.out_schema);
  }
  dbsp_schema out_schema() const override { return pj.out_schema; }
  orc_batch* step(Worker& w, const Slice&, const Slice&, const Slice& bid) override {
    orc_batch* bt = from_table(w, bid, pt);
    u64 k[DBSP_MAX_LANES];
    int32_t valid = 0;
    orc_batch_last_key(w.ctx, bt, k, &valid);
    if (valid) wm = std::max(wm, k[0] - 4000);                  // watermark_monotonic (q7.rs:60-61)
    wm = w.allreduce_max(wm);
    const u64 rounded = wm - (wm % 10000);                        // q7.rs:64-70
    u64 lo[DBSP_MAX_LANES] = {rounded >= 10000 ? rounded - 10000 : 0}, hi[DBSP_MAX_LANES] = {rounded};
    u64 plo[DBSP_MAX_LANES] = {has_prev ? prev_lo : lo[0]}, phi[DBSP_MAX_LANES] = {has_prev ? prev_hi : hi[0]};
    orc_batch* windowed = nullptr;
    orc_window_delta(w.ctx, wtrace, bt, has_prev ? 1 : 0, plo, phi, lo, hi, &windowed);
    orc_spine_insert(w.ctx, wtrace, bt);
    orc_spine_truncate_keys_below(w.ctx, wtrace, lo);
    orc_batch_free(bt);
    has_prev = true; prev_lo = lo[0]; prev_hi = hi[0];
    orc_batch* by_price = map_index(w, windowed, pprice, false);
    orc_batch* neg = map_index(w, windowed, pneg);
    if (w.T > 1) neg = aggregate_step(w, neg, loc_in, loc_out, DBSP_AGG_MIN);   // per-worker partial minima (min.rs:17-27)
    orc_batch* mp = map_index(w, aggregate_step(w, w.shard(neg), min_in, min_out, DBSP_AGG_MIN), pmax);
    orc_batch* bs[2] = {mp, by_price};
    w.shard_many(bs, 2);
    return join_step(w, bs[0], bs[1], lt, rt, pj);
  }
};

inline u64 mix64(u64 x) {
  x += 0x9e3779b97f4a7c15ull;
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}

// order-independent fingerprint of a Z-set: sum over tuples of hash(row) * weight (wrapping)
u64 fingerprint(Worker& w, orc_batch* b, const dbsp_schema& s, u64* n_out) {
  u64 n = 0, nkeys = 0;
  orc_batch_len(b, &n);
  *n_out = n;
  if (!n) return 0;
  orc_batch_key_count(w.ctx, b, &nkeys);
  const int nk = s.n_key_lanes, nv = s.n_val_lanes;
  std::vector<std::vector<u64>> keys((size_t)nk, std::vector<u64>(nkeys)), vals((size_t)nv, std::vector<u64>(n));
  std::vector<u64> offs(nkeys + 1);
  std::vector<i64> diffs(n);
  u64* kp[DBSP_MAX_LANES] = {nullptr};
  u64* vp[DBSP_MAX_LANES] = {nullptr};
  for (int l = 0; l < nk; l++) kp[l] = keys[(size_t)l].data();
  for (int l = 0; l < nv; l++) vp[l] = vals[(size_t)l].data();
  orc_batch_download_csr(w.ctx, b, kp, nv ? offs.data() : nullptr, vp, diffs.data());
  u64 fp = 0;
  for (u64 k = 0; k < nkeys; k++) {
    const u64 lo = nv ? offs[k] : k, hi = nv ? offs[k + 1] : k + 1;
    u64 hk = 0x243f6a8885a308d3ull;
    for (int l = 0; l < nk; l++) hk = mix64(hk ^ keys[(size_t)l][k]);
    for (u64 v = lo; v < hi; v++) {
      u64 h = hk;
      for (int l = 0; l < nv; l++) h = mix64(h ^ vals[(size_t)l][v]);
      fp += h * (u64)diffs[v];
    }
  }
  return fp;
}

}  // namespace

extern "C" {

// Runs `n_steps` steps of query `query` (3, 4, 7) on `n_threads` worker replicas.
//   cols   : [n_steps][3 tables: person, auction, bid][5] column pointers (NULL for tables the query ignores)
//   counts : [n_steps][3] row counts
// Worker r processes rows [r*n/T, (r+1)*n/T) of every table of the step.  Per step: wall seconds of the
// slowest worker (barrier to barrier), the gathered output's tuple count and fingerprint.
int32_t orcw_run(int32_t query, int32_t n_threads, int32_t n_steps, const u64* const* cols, const u64* counts,
                 double* step_seconds, u64* out_rows, u64* out_fp) {
  if (n_threads < 1 || (query != 3 && query != 4 && query != 7)) return DBSP_ERR_INVALID;
  Shared sh(n_threads);
  Barrier outer(n_threads);
  std::vector<std::thread> th;
  std::vector<std::chrono::steady_clock::time_point> t0((size_t)n_steps), t1((size_t)n_steps);
  for (int r = 0; r < n_threads; r++) {
    th.emplace_back([&, r] {
      Worker w;
      w.sh = &sh;
      w.rank = r;
      w.T = n_threads;
      orc_ctx_create(0, &w.ctx);
      Query* q = query == 3 ? (Query*)new Q3(w) : query == 4 ? (Query*)new Q4(w) : (Query*)new Q7(w);
      const dbsp_schema os = q->out_schema();
      for (int s = 0; s < n_steps; s++) {
        Slice sl[3];
        for (int t = 0; t < 3; t++) {
          const u64 n = counts[(size_t)s * 3 + t];
          const u64 lo = n * (u64)r / (u64)n_threads, hi = n * (u64)(r + 1) / (u64)n_threads;
          bool have = true;
          for (int c = 0; c < 5; c++) {
            const u64* p = cols[((size_t)s * 3 + t) * 5 + c];
            sl[t].cols[c] = p ? p + lo : nullptr;
            if (!p) have = false;
          }
          sl[t].n = have ? hi - lo : 0;
          if (!have) {   // table not materialised for this query: present empty columns
            static const u64 dummy = 0;
            for (int c = 0; c < 5; c++) sl[t].cols[c] = &dummy;
          }
        }
        outer.wait();
        if (r == 0) t0[(size_t)s] = std::chrono::steady_clock::now();
        orc_batch* out = q->step(w, sl[0], sl[1], sl[2]);
        outer.wait();
        if (r == 0) t1[(size_t)s] = std::chrono::steady_clock::now();
        // verification only (outside the timed interval): gather the output to worker 0
        orc_batch* g = w.gather0(out, os);
        if (r == 0) out_fp[s] = fingerprint(w, g, os, &out_rows[s]);
        orc_batch_free(g);
      }
    });
  }
  for (auto& t : th) t.join();
  for (int s = 0; s < n_steps; s++) step_seconds[s] = std::chrono::duration<double>(t1[(size_t)s] - t0[(size_t)s]).count();
  return DBSP_OK;
}

}  // extern "C"
