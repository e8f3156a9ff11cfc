// dbsp_oracle.cpp — CPU restatement of the reference's Z-set delta hot path.
//
// TEST INFRASTRUCTURE ONLY.  Nothing in the product package may link, load or
// call this file; only tests/, __graft_entry__.smoke() and bench.py's
// cpu_baseline / --impl reference legs use it, as the checker or as the timed
// CPU baseline.  The reference is Rust and cannot be built here (no rustc), so
// this is a "port": every routine follows the reference file:line it cites
// (paths relative to /root/reference/crates/dbsp/src/).  Parity is pinned by
// the reference's own golden vectors (tests/test_oracle_golden.py), see
// SURVEY.md §8c.
//
// The C entry points mirror include/dbsp_b200.h one to one with the prefix
// `orc_` so that the same host-side operator layer can be driven against the
// oracle from the test-suite.
//
// Storage follows the reference structs: OrdZSet = ColumnLayer{keys,diffs}
// (trace/ord/zset_batch.rs:28-31, trace/layers/column_layer/mod.rs:31-36);
// OrdIndexedZSet = OrderedLayer{keys,offs,ColumnLayer{vals,diffs}}
// (trace/ord/indexed_zset_batch.rs:27-41, trace/layers/ordered/mod.rs:32-44).

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../include/dbsp_b200.h"
#include "../database-stream-processor_b200/csrc/validate.h"

typedef uint64_t u64;
typedef int64_t i64;
#define MAXL DBSP_MAX_LANES

namespace {

// A column-major layer of `nl` lanes, `n` rows (nl may be 0: key = ()).
struct Layer {
  int nl = 0;
  uint8_t ty[MAXL] = {0};
  std::vector<u64> c[MAXL];
  size_t n = 0;
  void init(int nl_, const uint8_t* ty_) {
    nl = nl_;
    for (int l = 0; l < nl; l++) ty[l] = ty_[l];
  }
  void push(const u64* row) {
    for (int l = 0; l < nl; l++) c[l].push_back(row[l]);
    n++;
  }
  void push_from(const Layer& o, size_t i) {
    for (int l = 0; l < nl; l++) c[l].push_back(o.c[l][i]);
    n++;
  }
  void get(size_t i, u64* row) const {
    for (int l = 0; l < nl; l++) row[l] = c[l][i];
  }
};

inline int cmp1(uint8_t ty, u64 a, u64 b) {
  if (ty == DBSP_I64) return ((i64)a < (i64)b) ? -1 : ((i64)a > (i64)b);
  return (a < b) ? -1 : (a > b);
}
inline int cmp_rows(const Layer& A, size_t i, const Layer& B, size_t j) {
  for (int l = 0; l < A.nl; l++) {
    int c = cmp1(A.ty[l], A.c[l][i], B.c[l][j]);
    if (c) return c;
  }
  return 0;
}
inline int cmp_row_tuple(const Layer& A, size_t i, const u64* t) {
  for (int l = 0; l < A.nl; l++) {
    int c = cmp1(A.ty[l], A.c[l][i], t[l]);
    if (c) return c;
  }
  return 0;
}
inline int cmp_tuples(const uint8_t* ty, int nl, const u64* a, const u64* b) {
  for (int l = 0; l < nl; l++) {
    int c = cmp1(ty[l], a[l], b[l]);
    if (c) return c;
  }
  return 0;
}

struct Batch {
  dbsp_schema s;
  Layer K;                 // keys (n = key count; = tuple count when nv == 0)
  std::vector<u64> offs;   // nkeys+1 when nv > 0
  Layer V;                 // values (nv lanes)
  std::vector<i64> w;      // diffs
  explicit Batch(const dbsp_schema& sc) : s(sc) {
    K.init(s.n_key_lanes, s.lane_types);
    V.init(s.n_val_lanes, s.lane_types + s.n_key_lanes);
    if (s.n_val_lanes) offs.push_back(0);
  }
  bool indexed() const { return s.n_val_lanes > 0; }
  size_t len() const { return w.size(); }
  size_t nkeys() const { return K.n; }
  void vrange(size_t ki, size_t& lo, size_t& hi) const {
    if (indexed()) { lo = offs[ki]; hi = offs[ki + 1]; } else { lo = ki; hi = ki + 1; }
  }
};
typedef std::shared_ptr<Batch> BatchP;

// advance: count of the prefix of [lo,hi) satisfying the monotone predicate.
// Linear scan of <= 8, then exponential + binary search
// (trace/layers/advance.rs:3,25-72).
template <class F>
size_t advance(size_t lo, size_t hi, F pred) {
  const size_t SMALL = 8;
  size_t len = hi - lo;
  if (len > SMALL && pred(lo + SMALL)) {
    size_t index = SMALL + 1;
    if (index < len && pred(lo + index)) {
      size_t step = 1;
      while (index + step < len && pred(lo + index + step)) { index += step; step <<= 1; }
      step >>= 1;
      while (step > 0) {
        if (index + step < len && pred(lo + index + step)) index += step;
        step >>= 1;
      }
      index += 1;
    }
    return index;
  }
  size_t limit = std::min(len, SMALL);
  for (size_t i = 0; i < limit; i++) if (!pred(lo + i)) return i;
  return limit;
}

// Builder (trace/layers/ordered/mod.rs:468-479,874-888;
// column_layer/builders.rs:203-216): rows arrive sorted and consolidated.
struct Builder {
  BatchP b;
  explicit Builder(const dbsp_schema& s) : b(std::make_shared<Batch>(s)) {}
  void push(const u64* key, const u64* val, i64 w) {
    Batch& B = *b;
    if (!B.indexed()) { B.K.push(key); B.w.push_back(w); return; }
    if (B.K.n == 0 || cmp_row_tuple(B.K, B.K.n - 1, key) != 0) {
      if (B.K.n > 0) B.offs.push_back(B.w.size());  // close previous key
      B.K.push(key);
    }
    B.V.push(val);
    B.w.push_back(w);
  }
  BatchP done() {
    Batch& B = *b;
    if (B.indexed()) { if (B.K.n > 0) B.offs.push_back(B.w.size()); }
    return b;
  }
};

// consolidate (trace/consolidation/mod.rs:32-52,182-231): the tuples are gathered into an array of
// ((K,V),R) structs like the reference's Vec<((K,V),R)>, sorted by key, the weights of equal keys
// summed in place, zeros dropped; then Builder (merge_batcher/mod.rs:65-80).  The reference sorts with
// its own pdqsort (consolidation/quicksort.rs:12-33); only the sorted order is observable, std::sort
// (introsort) stands in.  i64 lanes are sorted through the order-preserving map x ^ 2^63.
template <int NL>
struct RowT {
  u64 k[NL];
  i64 w;
};
template <int NL>
BatchP from_tuples_n(const dbsp_schema& s, const u64* const* cols, const i64* w, size_t n) {
  typedef RowT<NL> Row;
  u64 flip[NL];
  for (int l = 0; l < NL; l++) flip[l] = s.lane_types[l] == DBSP_I64 ? 0x8000000000000000ull : 0ull;
  std::vector<Row> v(n);
  for (size_t i = 0; i < n; i++) {
    for (int l = 0; l < NL; l++) v[i].k[l] = cols[l][i] ^ flip[l];
    v[i].w = w ? w[i] : 1;
  }
  auto less = [](const Row& a, const Row& b) {
    for (int l = 0; l < NL; l++)
      if (a.k[l] != b.k[l]) return a.k[l] < b.k[l];
    return false;
  };
  auto same = [](const Row& a, const Row& b) {
    for (int l = 0; l < NL; l++)
      if (a.k[l] != b.k[l]) return false;
    return true;
  };
  std::sort(v.begin(), v.end(), less);
  Builder bld(s);
  u64 row[MAXL];
  size_t i = 0;
  while (i < n) {
    size_t j = i + 1;
    i64 sum = v[i].w;
    while (j < n && same(v[i], v[j])) {
      sum = (i64)((u64)sum + (u64)v[j].w);  // isize add wraps in release
      j++;
    }
    if (sum != 0) {
      for (int l = 0; l < NL; l++) row[l] = v[i].k[l] ^ flip[l];
      bld.push(row, row + s.n_key_lanes, sum);
    }
    i = j;
  }
  return bld.done();
}
BatchP from_tuples(const dbsp_schema& s, const u64* const* cols, const i64* w, size_t n) {
  switch (s.n_key_lanes + s.n_val_lanes) {
    case 1: return from_tuples_n<1>(s, cols, w, n);
    case 2: return from_tuples_n<2>(s, cols, w, n);
    case 3: return from_tuples_n<3>(s, cols, w, n);
    case 4: return from_tuples_n<4>(s, cols, w, n);
    case 5: return from_tuples_n<5>(s, cols, w, n);
    case 6: return from_tuples_n<6>(s, cols, w, n);
    case 7: return from_tuples_n<7>(s, cols, w, n);
    default: return from_tuples_n<8>(s, cols, w, n);
  }
}

// Tuple accumulator feeding from_tuples.
struct Tuples {
  dbsp_schema s;
  std::vector<u64> c[MAXL];
  std::vector<i64> w;
  explicit Tuples(const dbsp_schema& sc) : s(sc) {}
  void push(const u64* row, i64 wt) {
    int nl = s.n_key_lanes + s.n_val_lanes;
    for (int l = 0; l < nl; l++) c[l].push_back(row[l]);
    w.push_back(wt);
  }
  BatchP build() {
    const u64* cols[MAXL];
    for (int l = 0; l < MAXL; l++) cols[l] = c[l].data();
    return from_tuples(s, cols, w.data(), w.size());
  }
};

// ColumnLayerBuilder::copy_range + push_merge
// (trace/layers/column_layer/builders.rs:85-96, 98-169): galloping 2-way
// merge, copies capped at 1000 rows, equal keys summed, zero sums dropped.
void leaf_push_merge(Layer& outK, std::vector<i64>& outW, const Layer& A, const std::vector<i64>& wa,
                     size_t lo1, size_t hi1, const Layer& B, const std::vector<i64>& wb, size_t lo2,
                     size_t hi2) {
  auto copy_range = [&](const Layer& S, const std::vector<i64>& ws, size_t lo, size_t hi) {
    for (int l = 0; l < S.nl; l++) outK.c[l].insert(outK.c[l].end(), S.c[l].begin() + lo, S.c[l].begin() + hi);
    outK.n += hi - lo;
    outW.insert(outW.end(), ws.begin() + lo, ws.begin() + hi);
  };
  while (lo1 < hi1 && lo2 < hi2) {
    int c = cmp_rows(A, lo1, B, lo2);
    if (c < 0) {
      size_t step = 1 + advance(lo1 + 1, hi1, [&](size_t i) { return cmp_rows(A, i, B, lo2) < 0; });
      step = std::min<size_t>(step, 1000);
      copy_range(A, wa, lo1, lo1 + step);
      lo1 += step;
    } else if (c == 0) {
      i64 sum = (i64)((u64)wa[lo1] + (u64)wb[lo2]);
      if (sum != 0) { outK.push_from(A, lo1); outW.push_back(sum); }
      lo1++; lo2++;
    } else {
      size_t step = 1 + advance(lo2 + 1, hi2, [&](size_t i) { return cmp_rows(B, i, A, lo1) < 0; });
      step = std::min<size_t>(step, 1000);
      copy_range(B, wb, lo2, lo2 + step);
      lo2 += step;
    }
  }
  if (lo1 < hi1) copy_range(A, wa, lo1, hi1);
  if (lo2 < hi2) copy_range(B, wb, lo2, hi2);
}

// Merger (trace/mod.rs:371-396).  OrdZSet: one leaf push_merge, not fuelled
// (zset_batch.rs:307-318).  OrdIndexedZSet: OrderedBuilder::merge_step /
// push_merge_fueled / copy_range (trace/layers/ordered/mod.rs:344-396,
// 493-574, 787-834) and, with a lower value bound, the *_truncate_values_fueled
// variants (:587-746): on equal keys merge the two value ranges (seeked to the
// bound) and keep the key iff something survived; offsets rebased.  Fuel is
// counted in values produced; a merge whose call returns with fuel > 0 is
// complete (trace/mod.rs:378-395).
struct Merger {
  BatchP a, b, out;
  size_t lo1 = 0, hi1 = 0, lo2 = 0, hi2 = 0;
  Merger(BatchP a_, BatchP b_) : a(a_), b(b_), out(std::make_shared<Batch>(a_->s)) {
    hi1 = a->K.n;
    hi2 = b->K.n;
  }
  bool complete() const { return lo1 == hi1 && lo2 == hi2; }
  // first value index of key k of S that is >= the bound (cursor.seek(val_bound))
  static size_t vstart(const Batch& S, size_t k, const u64* vb) {
    size_t vlo = S.offs[k], vhi = S.offs[k + 1];
    if (!vb) return vlo;
    return vlo + advance(vlo, vhi, [&](size_t i) { return cmp_row_tuple(S.V, i, vb) < 0; });
  }
  // copy_range[_truncate_values]_fueled (ordered/mod.rs:541-574, 711-746)
  size_t copy_range(const Batch& S, size_t lo, size_t hi, const u64* vb, size_t fuel) {
    Batch& O = *out;
    size_t start = S.offs[lo];
    for (size_t k = lo; k < hi; k++) {
      size_t vlo = vstart(S, k, vb), vhi = S.offs[k + 1];
      if (vhi > vlo) {
        O.K.push_from(S.K, k);
        for (int l = 0; l < S.V.nl; l++) O.V.c[l].insert(O.V.c[l].end(), S.V.c[l].begin() + vlo, S.V.c[l].begin() + vhi);
        O.V.n += vhi - vlo;
        O.w.insert(O.w.end(), S.w.begin() + vlo, S.w.begin() + vhi);
        O.offs.push_back(O.w.size());
      }
      if (vhi - start >= fuel) return k + 1;
    }
    return hi;
  }
  void merge_step(const u64* vb) {
    const Batch &A = *a, &B = *b;
    Batch& O = *out;
    int c = cmp_rows(A.K, lo1, B.K, lo2);
    if (c < 0) {
      size_t step = 1 + advance(lo1 + 1, hi1, [&](size_t i) { return cmp_rows(A.K, i, B.K, lo2) < 0; });
      step = std::min<size_t>(step, 1000);
      lo1 = copy_range(A, lo1, lo1 + step, vb, SIZE_MAX);
    } else if (c == 0) {
      size_t before = O.w.size();
      leaf_push_merge(O.V, O.w, A.V, A.w, vstart(A, lo1, vb), A.offs[lo1 + 1], B.V, B.w, vstart(B, lo2, vb), B.offs[lo2 + 1]);
      if (O.w.size() > before) { O.K.push_from(A.K, lo1); O.offs.push_back(O.w.size()); }
      lo1++; lo2++;
    } else {
      size_t step = 1 + advance(lo2 + 1, hi2, [&](size_t i) { return cmp_rows(B.K, i, A.K, lo1) < 0; });
      step = std::min<size_t>(step, 1000);
      lo2 = copy_range(B, lo2, lo2 + step, vb, SIZE_MAX);
    }
  }
  void work(const u64* vb, i64* fuel) {
    Batch& O = *out;
    if (!a->indexed()) {   // zset_batch.rs:307-318: whole merge, fuel clamped to >= 1
      size_t before = O.w.size();
      leaf_push_merge(O.K, O.w, a->K, a->w, lo1, hi1, b->K, b->w, lo2, hi2);
      lo1 = hi1; lo2 = hi2;
      *fuel -= (i64)(O.w.size() - before);
      *fuel = std::max<i64>(*fuel, 1);
      return;
    }
    size_t starting = O.w.size();
    i64 effort = 0;
    while (lo1 < hi1 && lo2 < hi2 && effort < *fuel) {
      merge_step(vb);
      effort = (i64)(O.w.size() - starting);
    }
    if (lo1 == hi1 || lo2 == hi2) {
      i64 remaining = *fuel - effort;
      if (remaining > 0) {
        if (lo1 < hi1) { if (remaining < 1000) remaining = 1000; lo1 = copy_range(*a, lo1, hi1, vb, (size_t)remaining); }
        if (lo2 < hi2) { if (remaining < 1000) remaining = 1000; lo2 = copy_range(*b, lo2, hi2, vb, (size_t)remaining); }
      }
    }
    effort = (i64)(O.w.size() - starting);
    *fuel -= effort;
  }
};

// Batch::merge = Merger run to completion (trace/mod.rs:280-291).
BatchP merge(const BatchP& a, const BatchP& b, const u64* vb = nullptr) {
  Merger m(a, b);
  while (!m.complete()) {
    i64 fuel = INT64_MAX;
    m.work(vb, &fuel);
  }
  return m.out;
}

// Cursor::seek_key: first key index >= `key` (exponential search from `from`,
// trace/layers/column_layer/cursor.rs:121-128 via advance).
size_t seek_key(const Batch& b, size_t from, const u64* key) {
  return from + advance(from, b.K.n, [&](size_t i) { return cmp_row_tuple(b.K, i, key) < 0; });
}

// truncate_keys_below (column_layer/mod.rs:316-319, trace/mod.rs:227-233):
// the reference only raises `lower_bound`; cursors start there.  The oracle
// materialises the suffix, which is observably the same.
BatchP truncate_keys_below(const Batch& b, const u64* key) {
  size_t k0 = seek_key(b, 0, key);
  if (k0 == 0) return nullptr;
  auto out = std::make_shared<Batch>(b.s);
  Batch& O = *out;
  for (size_t k = k0; k < b.K.n; k++) {
    O.K.push_from(b.K, k);
    size_t lo, hi;
    b.vrange(k, lo, hi);
    if (b.indexed()) {
      for (size_t v = lo; v < hi; v++) { O.V.push_from(b.V, v); O.w.push_back(b.w[v]); }
      O.offs.push_back(O.w.size());
    } else {
      O.w.push_back(b.w[k]);
    }
  }
  return out;
}

// Spine (trace/spine_fueled.rs:107-119).  The reference places a batch at
// level log2(len.next_power_of_two()) and spends fuel on in-progress merges
// (:605-634, :730-812).  The merge *schedule* is unobservable in operator
// outputs (cursors see the union of all batches, cursor/cursor_list.rs), so
// this oracle — like the CUDA spine — keeps the same geometric invariant with
// eager merges: after an insert, while the two newest batches are within 2x
// of each other they are merged.  Documented in DESIGN.md.
// Spine (trace/spine_fueled.rs:107-119, 537-1188): the fuelled LSM, restated layer by layer.  `merging[i]`
// is MergeState of layer i; a merge in progress keeps both inputs visible to cursors (:179-216) while the
// Merger (above) advances by the fuel every insert grants it.  `batches` is the cursor view, rebuilt after
// every mutation.
struct Spine {
  struct Layer {
    enum Kind { VACANT, SINGLE, IN_PROGRESS, COMPLETE } kind = VACANT;
    BatchP a, b;                     // SINGLE: a (may be null = structurally empty); IN_PROGRESS: a, b; COMPLETE: a (may be null)
    std::shared_ptr<Merger> m;       // IN_PROGRESS
    size_t len() const {             // MergeState::len (:1034-1041)
      switch (kind) {
        case SINGLE: case COMPLETE: return a ? a->len() : 0;
        case IN_PROGRESS: return a->len() + b->len();
        default: return 0;
      }
    }
    bool is_double() const { return kind == IN_PROGRESS || kind == COMPLETE; }
  };
  dbsp_schema s;
  std::vector<Layer> merging;
  std::vector<BatchP> batches;   // cursor view, largest layer first
  size_t effort = 1;
  bool has_bound = false;
  u64 bound[MAXL] = {};   // zero until set: spine_save writes both arrays whole
  bool has_vbound = false;   // lower_val_bound (spine_fueled.rs:118, 644-656)
  u64 vbound[MAXL] = {};
  explicit Spine(const dbsp_schema& sc) : s(sc) {}
  const u64* vb() const { return has_vbound ? vbound : nullptr; }

  void refresh() {
    batches.clear();
    for (size_t i = merging.size(); i-- > 0;) {
      const Layer& l = merging[i];
      if (l.kind == Layer::IN_PROGRESS) {
        if (l.a->len()) batches.push_back(l.a);
        if (l.b->len()) batches.push_back(l.b);
      } else if ((l.kind == Layer::SINGLE || l.kind == Layer::COMPLETE) && l.a && l.a->len()) {
        batches.push_back(l.a);
      }
    }
  }
  static Layer begin_merge(BatchP b1, BatchP b2) {   // MergeState::begin_merge (:1106-1124)
    Layer l;
    if (b1 && b2) {
      l.kind = Layer::IN_PROGRESS;
      l.a = b1;
      l.b = b2;
      l.m = std::make_shared<Merger>(b1, b2);
    } else {
      l.kind = Layer::COMPLETE;
      l.a = b1 ? b1 : b2;
    }
    return l;
  }
  void work(Layer& l, i64* fuel) {   // MergeVariant::work (:1176-1188)
    if (l.kind != Layer::IN_PROGRESS) return;
    l.m->work(vb(), fuel);
    if (*fuel > 0) {
      if (!l.m->complete()) {   // fuel left although the inputs are not exhausted cannot happen for a fuelled merger
        i64 more = INT64_MAX;
        while (!l.m->complete()) l.m->work(vb(), &more);
      }
      l.kind = Layer::COMPLETE;
      l.a = l.m->out;
      l.b = nullptr;
      l.m = nullptr;
    }
  }
  BatchP complete(Layer& l) {   // MergeState::complete (:1060-1066)
    BatchP r;
    if (l.kind == Layer::IN_PROGRESS) {
      while (l.kind == Layer::IN_PROGRESS) { i64 fuel = INT64_MAX; work(l, &fuel); }
    }
    if (l.kind == Layer::SINGLE || l.kind == Layer::COMPLETE) r = l.a;
    l = Layer();
    return r;
  }
  void insert_at(BatchP batch, size_t index) {   // (:889-908)
    while (merging.size() <= index) merging.push_back(Layer());
    Layer& l = merging[index];
    if (l.kind == Layer::VACANT) { l.kind = Layer::SINGLE; l.a = batch; }
    else if (l.kind == Layer::SINGLE) { BatchP old = l.a; l = begin_merge(old, batch); }
    else { fprintf(stderr, "oracle spine: attempted to insert a batch into an incomplete merge\n"); abort(); }   // panic! (:904)
  }
  void apply_fuel(i64 fuel_each) {   // (:856-882)
    for (size_t index = 0; index < merging.size(); index++) {
      i64 fuel = fuel_each;
      work(merging[index], &fuel);
      if (merging[index].kind == Layer::COMPLETE) {
        BatchP done = complete(merging[index]);
        insert_at(done, index + 1);
      }
    }
  }
  void roll_up(size_t index) {   // (:819-846)
    while (merging.size() <= index) merging.push_back(Layer());
    bool any = false;
    for (size_t i = 0; i < index; i++) any = any || merging[i].kind != Layer::VACANT;
    if (!any) return;
    BatchP merged;
    for (size_t i = 0; i < index; i++) {
      insert_at(merged, i);
      merged = complete(merging[i]);
    }
    insert_at(merged, index);
    if (merging[index].is_double()) {
      BatchP m2 = complete(merging[index]);
      insert_at(m2, index + 1);
    }
  }
  void tidy_layers() {   // (:916-974)
    if (merging.empty()) return;
    size_t length = merging.size();
    if (merging[length - 1].kind != Layer::SINGLE) return;
    size_t len = merging[length - 1].len(), appropriate = 0;
    while (((size_t)1 << appropriate) < len) appropriate++;
    while (appropriate < length - 1) {
      Layer& below = merging[length - 2];
      if (below.kind == Layer::VACANT || (below.kind == Layer::SINGLE && !below.a)) {
        merging.erase(merging.begin() + (length - 2));
        length = merging.size();
      } else if (below.kind == Layer::SINGLE) {
        u64 smaller = 0;
        for (size_t i = 0; i + 2 < length; i++) {
          if (merging[i].kind == Layer::SINGLE) smaller += 1ull << i;
          else if (merging[i].is_double()) smaller += 2ull << i;
        }
        if (smaller <= (1ull << length) / 8) {
          BatchP batch = below.a;
          merging.erase(merging.begin() + (length - 2));
          insert_at(batch, length - 2);
        }
        return;
      } else {
        return;
      }
    }
  }
  void introduce_batch(BatchP batch, size_t batch_index) {   // (:728-812)
    i64 fuel = batch_index >= 59 ? INT64_MAX : (i64)((8ull << batch_index) * effort);
    apply_fuel(fuel);
    roll_up(batch_index);
    insert_at(batch, batch_index);
    tidy_layers();
  }
  bool reduced() const {   // (:663-680)
    int non_empty = 0;
    for (const Layer& l : merging) {
      if (l.is_double()) return false;
      if (l.len() > 0) non_empty++;
      if (non_empty > 1) return false;
    }
    return true;
  }
  void insert(BatchP b) {   // Trace::insert (:605-634)
    if (b->len() == 0) return;
    if (has_bound) { BatchP t = truncate_keys_below(*b, bound); if (t) b = t; }
    size_t index = 0;
    while (((size_t)1 << index) < b->len()) index++;
    introduce_batch(b, index);
    refresh();
  }
  void exert(i64* effort_) {   // Trace::exert (:561-581)
    tidy_layers();
    if (!reduced()) {
      bool any_double = false;
      for (const Layer& l : merging) any_double = any_double || l.is_double();
      if (any_double) apply_fuel(*effort_);
      else {
        size_t level = 0;
        while ((1ull << level) < (u64)(*effort_ > 0 ? *effort_ : 1) && level < 62) level++;
        introduce_batch(nullptr, level);
      }
    }
    refresh();
  }
  // A consolidated read of the trace: the merge of everything a cursor sees, the value bound applied.
  // (Trace::consolidate (:583-600) consumes the trace; this leaves the layers as they are.)
  BatchP consolidate() {
    BatchP acc = std::make_shared<Batch>(s);
    for (auto& b : batches) acc = merge(acc, b, vb());
    return acc;
  }
  void truncate(const u64* key) {   // truncate_keys_below (:223-233)
    if (has_bound && cmp_tuples(s.lane_types, s.n_key_lanes, key, bound) <= 0) return;   // bound = max(old, new)
    for (Layer& l : merging) { i64 fuel = INT64_MAX; while (l.kind == Layer::IN_PROGRESS) work(l, &fuel); }   // complete_merges (:977-985)
    has_bound = true;
    for (int l = 0; l < s.n_key_lanes; l++) bound[l] = key[l];
    for (Layer& l : merging) {   // map_batches_mut (:988-1004)
      if ((l.kind == Layer::SINGLE || l.kind == Layer::COMPLETE) && l.a) {
        BatchP t = truncate_keys_below(*l.a, bound);
        if (t) l.a = t;
      }
    }
    refresh();
  }
  // truncate_values_below (spine_fueled.rs:644-652): the bound only grows; it is
  // applied by later merges (:866, :911, :981), contents below it are undefined.
  void truncate_values(const u64* val) {
    const uint8_t* ty = s.lane_types + s.n_key_lanes;
    if (!has_vbound || cmp_tuples(ty, s.n_val_lanes, val, vbound) > 0)
      for (int l = 0; l < s.n_val_lanes; l++) vbound[l] = val[l];
    has_vbound = true;
  }
  size_t len() const { size_t n = 0; for (auto& b : batches) n += b->len(); return n; }
};

// CursorList view of one key (trace/cursor/cursor_list.rs:57-127,200-210):
// the union of the key's values over all spine batches in value order, the
// weight of a value being the SUM over batches (may be zero).
struct KV { const Batch* b; size_t pos; };
void key_group(const Spine& sp, const u64* key, std::vector<std::pair<KV, i64>>& out) {
  out.clear();
  std::vector<KV> all;
  for (auto& bp : sp.batches) {
    const Batch& b = *bp;
    size_t k = seek_key(b, 0, key);
    if (k < b.K.n && cmp_row_tuple(b.K, k, key) == 0) {
      size_t lo, hi;
      b.vrange(k, lo, hi);
      for (size_t v = lo; v < hi; v++) all.push_back({&b, v});
    }
  }
  std::stable_sort(all.begin(), all.end(), [](const KV& x, const KV& y) {
    return x.b->V.nl && cmp_rows(x.b->V, x.pos, y.b->V, y.pos) < 0;
  });
  size_t i = 0;
  while (i < all.size()) {
    size_t j = i;
    i64 sum = 0;
    while (j < all.size() && (all[i].b->V.nl == 0 || cmp_rows(all[i].b->V, all[i].pos, all[j].b->V, all[j].pos) == 0)) {
      sum = (i64)((u64)sum + (u64)all[j].b->w[all[j].pos]);
      j++;
    }
    out.push_back({all[i], sum});
    i = j;
  }
}

// ---- declarative row expressions -------------------------------------
struct Env { const u64* key; const u64* lv; const u64* rv; };
inline u64 src_val(const dbsp_src& s, const Env& e) {
  switch (s.kind) {
    case DBSP_SRC_KEY: return e.key[s.idx];
    case DBSP_SRC_LVAL: return e.lv[s.idx];
    case DBSP_SRC_RVAL: return e.rv[s.idx];
    default: return (u64)s.cst;
  }
}
inline u64 expr_val(const dbsp_expr& x, const Env& e) {
  u64 a = src_val(x.a, e);
  switch (x.op) {
    case DBSP_OP_COPY: return a;
    case DBSP_OP_NEG: return (u64)0 - a;
    case DBSP_OP_ADD: return a + src_val(x.b, e);
    case DBSP_OP_SUB: return a - src_val(x.b, e);
    case DBSP_OP_MUL: return a * src_val(x.b, e);
    case DBSP_OP_DIV: {   // i64::wrapping_div, x / 0 = 0 (the ABI's rules; Rust's `/` panics on both)
      i64 d = (i64)src_val(x.b, e);
      if (d == 0) return 0;
      if (d == -1) return (u64)0 - a;   // MIN / -1 = MIN; the C++ division would trap
      return (u64)((i64)a / d);
    }
  }
  return a;
}
inline bool pred_ok(const dbsp_pred& p, const Env& e) {
  u64 a = src_val(p.a, e), b = src_val(p.b, e);
  int c = p.is_signed ? (((i64)a < (i64)b) ? -1 : ((i64)a > (i64)b)) : ((a < b) ? -1 : (a > b));
  switch (p.cmp) {
    case DBSP_CMP_EQ: return c == 0;
    case DBSP_CMP_NE: return c != 0;
    case DBSP_CMP_LT: return c < 0;
    case DBSP_CMP_LE: return c <= 0;
    case DBSP_CMP_GT: return c > 0;
    case DBSP_CMP_GE: return c >= 0;
    case DBSP_CMP_IN: return a < 64 && ((b >> a) & 1);
  }
  return false;
}
inline bool project(const dbsp_proj& p, const Env& e, u64* row) {
  for (int i = 0; i < p.n_pred; i++) if (!pred_ok(p.pred[i], e)) return false;
  int nl = p.out_schema.n_key_lanes + p.out_schema.n_val_lanes;
  for (int l = 0; l < nl; l++) row[l] = expr_val(p.out[l], e);
  return true;
}

// Join::eval (operator/join.rs:436-473) — also the inner loop of
// JoinTrace::eval (:751-787): merge-walk both key sets, on equal keys the
// cartesian product of the value ranges, weight = w1*w2 (MulByRef,
// algebra/mod.rs:195-213), join_func = proj.
void join_into(const Batch& L, const Batch& R, const dbsp_proj& proj, bool swap, Tuples& out) {
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
          if (project(proj, e, row)) out.push(row, (i64)((u64)L.w[a] * (u64)R.w[b]));
        }
      }
      i++; j++;
    }
  }
}

}  // namespace

// ===================== C entry points (prefix orc_) ======================
struct orc_batch { BatchP p; };
struct orc_spine { Spine s; explicit orc_spine(const dbsp_schema& sc) : s(sc) {} };
struct orc_ctx { int dummy; };
static thread_local std::string g_err;

static orc_batch* wrap(BatchP p) { return new orc_batch{p}; }

// The error contract of include/dbsp_b200.h: every argument is checked, by the call's check in validate.h (the CUDA
// library's), before the call reads or builds anything.  WHAT is the call's name without the prefix.
namespace dv = dbsp_validate;
#define WHAT (__func__ + 4)
#define REFUSE(check)                                       \
  do {                                                      \
    const dv::Refusal r__ = (check);                        \
    if (r__) { g_err = r__.text; return r__.status; }       \
  } while (0)
#define NOT_NULL(p, name) REFUSE(dv::not_null(p, WHAT, name))
// a handle's schema as the checks of validate.h take it: NULL for a NULL handle
static const dbsp_schema* S(const orc_batch* b) { return b ? &b->p->s : nullptr; }
static const dbsp_schema* S(const orc_spine* s) { return s ? &s->s.s : nullptr; }

extern "C" {

int32_t orc_ctx_create(int32_t device, orc_ctx** out) {
  REFUSE(dv::check_ctx_create(out, device));
  *out = new orc_ctx{0};
  return DBSP_OK;
}
int32_t orc_ctx_destroy(orc_ctx* c) { delete c; return DBSP_OK; }
int32_t orc_ctx_sync(orc_ctx* c) { NOT_NULL(c, "ctx"); return DBSP_OK; }
const char* orc_last_error(void) { return g_err.c_str(); }
int32_t orc_ctx_stats(orc_ctx* ctx, u64* a, u64* b, u64* c, int32_t) { NOT_NULL(ctx, "ctx"); if (a) *a = 0; if (b) *b = 0; if (c) *c = 0; return DBSP_OK; }
void* orc_ctx_stream(orc_ctx*) { return nullptr; }
int32_t orc_ctx_profile(orc_ctx* c, int32_t enable) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_ctx_profile(enable));
  return DBSP_OK;
}
int32_t orc_ctx_profile_read(orc_ctx*, int32_t, char*, u64*, double*, u64*) { return DBSP_ERR_INVALID; }

int32_t orc_batch_from_tuples(orc_ctx* c, const dbsp_schema* s, const u64* const* cols, const i64* w, u64 n,
                              int32_t, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_tuples(WHAT, out, s, cols, w, n, false));
  *out = wrap(from_tuples(*s, cols, w, n));
  return DBSP_OK;
}

// FlatMap::eval + from_tuples (operator/filter_map.rs:700-724).
static void table_to_batch(const u64* const* cols, uint32_t ncols, const i64* w, u64 n, const dbsp_proj* proj, orc_batch** out) {
  const unsigned used = dv::proj_table_mask(*proj);
  Tuples t(proj->out_schema);
  u64 lv[MAXL] = {0}, row[MAXL];
  for (u64 i = 0; i < n; i++) {
    for (uint32_t c = 0; c < ncols; c++) if ((used >> c) & 1) lv[c] = cols[c][i];
    Env e{lv, lv, lv};
    if (project(*proj, e, row)) t.push(row, w ? w[i] : 1);
  }
  *out = wrap(t.build());
}
int32_t orc_batch_from_table(orc_ctx* c, const u64* const* cols, uint32_t ncols, const i64* w, u64 n, int32_t,
                             const dbsp_proj* proj, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_table(WHAT, out, cols, ncols, n, proj));
  table_to_batch(cols, ncols, w, n, proj, out);
  return DBSP_OK;
}

// pipelined ingest: on the CPU there is nothing to overlap, keep the pointers
struct orc_upload { const orc_ctx* ctx; const u64* const* cols; uint32_t n_cols; uint32_t col_mask; const i64* w; u64 n; std::vector<const u64*> own; };
static dv::Upload upload_of(const orc_upload* u, const orc_ctx* c) {
  if (!u) return dv::Upload{false, false, 0, 0, 0};
  return dv::Upload{true, u->ctx == c, (int)u->n_cols, u->col_mask, u->n};
}
int32_t orc_upload_begin(orc_ctx* c, const u64* const* cols, uint32_t n_cols, uint32_t col_mask, const i64* w, u64 n, orc_upload** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_upload_begin(out, cols, n_cols, col_mask, n));
  orc_upload* u = new orc_upload();
  u->own.assign(cols, cols + n_cols);
  u->ctx = c; u->cols = u->own.data(); u->n_cols = n_cols; u->col_mask = col_mask; u->w = w; u->n = n;
  *out = u;
  return DBSP_OK;
}
int32_t orc_batch_from_upload(orc_ctx* c, orc_upload* u, const dbsp_proj* proj, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_upload(WHAT, out, upload_of(u, c), proj));
  table_to_batch(u->cols, u->n_cols, u->w, u->n, proj, out);
  return DBSP_OK;
}
int32_t orc_upload_free(orc_upload* u) { delete u; return DBSP_OK; }
uint32_t orc_proj_table_mask(const dbsp_proj* proj) { return dv::checked_table_mask(proj, WHAT); }

int32_t orc_batch_empty(orc_ctx* c, const dbsp_schema* s, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_new(WHAT, out, s));
  *out = wrap(std::make_shared<Batch>(*s));
  return DBSP_OK;
}

int32_t orc_batch_merge(orc_ctx* c, const orc_batch* a, const orc_batch* b, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_merge(WHAT, out, S(a), S(b)));
  *out = wrap(merge(a->p, b->p));
  return DBSP_OK;
}

// MergeBatcher (trace/ord/merge_batcher/mod.rs:22-81, 155-260): push consolidates
// and queues; the two newest entries merge while the newer is at least half the
// older (the reference counts 8 KiB chunks, this port counts rows); seal =
// finish_into + Builder.
struct orc_batcher { dbsp_schema s; std::vector<BatchP> queue; };
static void batcher_enqueue(orc_batcher* q, BatchP b) {
  if (b->len() == 0) return;
  q->queue.push_back(b);
  while (q->queue.size() > 1 && q->queue[q->queue.size() - 1]->len() >= q->queue[q->queue.size() - 2]->len() / 2) {
    BatchP y = q->queue.back(); q->queue.pop_back();
    BatchP x = q->queue.back(); q->queue.pop_back();
    BatchP m = merge(x, y);
    if (m->len()) q->queue.push_back(m);
  }
}
int32_t orc_batcher_new(orc_ctx* c, const dbsp_schema* s, orc_batcher** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_new(WHAT, out, s));
  *out = new orc_batcher{*s, {}};
  return DBSP_OK;
}
int32_t orc_batcher_push(orc_ctx* c, orc_batcher* q, const u64* const* cols, const i64* w, u64 n, int32_t) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_push(WHAT, q ? &q->s : nullptr, cols, w, n, false));
  if (n) batcher_enqueue(q, from_tuples(q->s, cols, w, n));
  return DBSP_OK;
}
int32_t orc_batch_from_sorted(orc_ctx* c, const dbsp_schema* s, const u64* const* cols, const i64* w, u64 n, int32_t od,
                              orc_batch** out);
int32_t orc_batcher_push_consolidated(orc_ctx* c, orc_batcher* q, const u64* const* cols, const i64* w, u64 n, int32_t od) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_push(WHAT, q ? &q->s : nullptr, cols, w, n, true));
  if (!n) return DBSP_OK;
  orc_batch* b = nullptr;
  int32_t rc = orc_batch_from_sorted(c, &q->s, cols, w, n, od, &b);
  if (rc) return rc;
  batcher_enqueue(q, b->p);
  delete b;
  return DBSP_OK;
}
int32_t orc_batcher_tuples(const orc_batcher* q, u64* n) { NOT_NULL(q, "batcher"); NOT_NULL(n, "n_tuples"); u64 t = 0; for (auto& b : q->queue) t += b->len(); *n = t; return DBSP_OK; }
int32_t orc_batcher_free(orc_batcher* q) { delete q; return DBSP_OK; }
int32_t orc_batcher_seal(orc_ctx* c, orc_batcher* q, orc_batch** out) {
  NOT_NULL(c, "ctx");
  NOT_NULL(q, "batcher");
  NOT_NULL(out, "out");
  while (q->queue.size() >= 2) {
    BatchP y = q->queue.back(); q->queue.pop_back();
    BatchP x = q->queue.back(); q->queue.pop_back();
    BatchP m = merge(x, y);
    if (m->len()) q->queue.push_back(m);
  }
  *out = wrap(q->queue.empty() ? std::make_shared<Batch>(q->s) : q->queue.back());
  delete q;
  return DBSP_OK;
}

// Merger::work with a lower value bound run to completion
// (indexed_zset_batch.rs:359-382; ordered/mod.rs:587-746).  OrdZSet ignores the
// bound (zset_batch.rs:307-318).
int32_t orc_batch_merge_bounded(orc_ctx* c, const orc_batch* a, const orc_batch* b, const u64* vb, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_merge(WHAT, out, S(a), S(b)));
  *out = wrap(merge(a->p, b->p, a->p->indexed() ? vb : nullptr));
  return DBSP_OK;
}
struct orc_merger { Merger m; bool has_vb; u64 vb[MAXL]; };
int32_t orc_merger_new(orc_ctx* c, const orc_batch* a, const orc_batch* b, const u64* vb, orc_merger** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_merge(WHAT, out, S(a), S(b)));
  orc_merger* m = new orc_merger{Merger(a->p, b->p), vb != nullptr && a->p->indexed(), {0}};
  if (m->has_vb) for (int l = 0; l < a->p->s.n_val_lanes; l++) m->vb[l] = vb[l];
  *out = m;
  return DBSP_OK;
}
int32_t orc_merger_work(orc_ctx* c, orc_merger* m, i64* fuel) {
  NOT_NULL(c, "ctx");
  NOT_NULL(m, "merger");
  NOT_NULL(fuel, "fuel");
  if (m->m.complete()) { *fuel = std::max<i64>(*fuel, 1); return DBSP_OK; }
  if (*fuel > 0) m->m.work(m->has_vb ? m->vb : nullptr, fuel);
  if (m->m.complete()) *fuel = std::max<i64>(*fuel, 1);   // ABI: fuel > 0 after the call <=> merge complete
  else *fuel = std::min<i64>(*fuel, 0);
  return DBSP_OK;
}
int32_t orc_merger_done(orc_ctx* c, orc_merger* m, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_merger_done(m, m && m->m.complete(), out));
  *out = wrap(m->m.out);
  delete m;
  return DBSP_OK;
}
int32_t orc_merger_free(orc_merger* m) { delete m; return DBSP_OK; }
// BatchReader::truncate_keys_below (trace/mod.rs:227-233).
int32_t orc_batch_truncate_keys_below(orc_ctx* c, const orc_batch* b, const u64* key, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_truncate(out, S(b), key));
  BatchP t = truncate_keys_below(*b->p, key);
  *out = wrap(t ? t : b->p);
  return DBSP_OK;
}

// neg (column_layer/mod.rs:452-480).
int32_t orc_batch_neg(orc_ctx* c, const orc_batch* a, orc_batch** out) {
  NOT_NULL(c, "ctx");
  NOT_NULL(out, "out");
  NOT_NULL(a, "batch");
  auto o = std::make_shared<Batch>(*a->p);
  for (auto& x : o->w) x = (i64)((u64)0 - (u64)x);
  *out = wrap(o);
  return DBSP_OK;
}

// Flat rows of a batch: (key lanes, val lanes, weight) per tuple.
static void flat_rows(const Batch& b, Tuples& t) {
  u64 row[MAXL];
  for (size_t k = 0; k < b.K.n; k++) {
    b.K.get(k, row);
    size_t lo, hi;
    b.vrange(k, lo, hi);
    for (size_t v = lo; v < hi; v++) {
      if (b.indexed()) b.V.get(v, row + b.s.n_key_lanes);
      t.push(row, b.w[v]);
    }
  }
}

// index() (operator/index.rs:128-157) and its inverse: re-split the lanes.
int32_t orc_batch_reindex(orc_ctx* c, const orc_batch* a, uint32_t nk, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_reindex(out, S(a), nk));
  dbsp_schema s = a->p->s;
  int nl = s.n_key_lanes + s.n_val_lanes;
  s.n_key_lanes = nk; s.n_val_lanes = nl - nk;
  Tuples t(s);
  flat_rows(*a->p, t);
  *out = wrap(t.build());
  return DBSP_OK;
}

int32_t orc_batch_len(const orc_batch* b, u64* n) { NOT_NULL(b, "batch"); NOT_NULL(n, "n_tuples"); *n = b->p->len(); return DBSP_OK; }
int32_t orc_batch_key_count(orc_ctx* c, const orc_batch* b, u64* n) {
  NOT_NULL(c, "ctx");
  NOT_NULL(b, "batch");
  NOT_NULL(n, "n_keys");
  *n = b->p->nkeys();
  return DBSP_OK;
}
int32_t orc_batch_schema(const orc_batch* b, dbsp_schema* out) { NOT_NULL(b, "batch"); NOT_NULL(out, "out"); *out = b->p->s; return DBSP_OK; }

int32_t orc_batch_download_csr(orc_ctx* c, const orc_batch* bb, u64* const* keys, u64* offs, u64* const* vals,
                               i64* diffs) {
  NOT_NULL(c, "ctx");
  NOT_NULL(bb, "batch");
  const Batch& b = *bb->p;
  if (keys) for (int l = 0; l < b.K.nl; l++) if (keys[l]) std::copy(b.K.c[l].begin(), b.K.c[l].end(), keys[l]);
  if (offs && b.indexed()) {
    if (b.K.n == 0) offs[0] = 0; else std::copy(b.offs.begin(), b.offs.end(), offs);
  }
  if (vals) for (int l = 0; l < b.V.nl; l++) if (vals[l]) std::copy(b.V.c[l].begin(), b.V.c[l].end(), vals[l]);
  if (diffs) std::copy(b.w.begin(), b.w.end(), diffs);
  return DBSP_OK;
}

int32_t orc_batch_device_columns(const orc_batch*, const u64**, const i64**) { return DBSP_ERR_UNSUPPORTED; }
// no device, no asynchronous reads: the oracle's outputs are compared through download_csr
struct orc_download;
int32_t orc_batch_download_begin(orc_ctx*, const orc_batch*, u64* const*, i64*, orc_download**) { return DBSP_ERR_UNSUPPORTED; }
int32_t orc_download_finish(orc_download*) { return DBSP_OK; }
int32_t orc_ctx_sync_stats(orc_ctx* c, u64* n, double* us, int32_t) { NOT_NULL(c, "ctx"); if (n) *n = 0; if (us) *us = 0; return DBSP_OK; }

// fast_forward_keys + get_key (operator/time_series/watermark.rs:38-45).
int32_t orc_batch_last_key(orc_ctx* c, const orc_batch* b, u64* key, int32_t* valid) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_last_key(S(b), key, valid));
  const Batch& B = *b->p;
  *valid = B.K.n > 0;
  if (B.K.n) B.K.get(B.K.n - 1, key);
  return DBSP_OK;
}
int32_t orc_batch_clone(const orc_batch* b, orc_batch** out) { NOT_NULL(b, "batch"); NOT_NULL(out, "out"); *out = wrap(b->p); return DBSP_OK; }
int32_t orc_batch_free(orc_batch* b) { delete b; return DBSP_OK; }

// Builder::push ... done (trace/mod.rs:338-368; ordered/mod.rs:468-479,874-888): the rows are already
// sorted and consolidated — appended in order, no sort.
int32_t orc_batch_from_sorted(orc_ctx* c, const dbsp_schema* s, const u64* const* cols, const i64* w, u64 n,
                              int32_t, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_tuples(WHAT, out, s, cols, w, n, true));
  Builder bld(*s);
  const int nk = s->n_key_lanes, nv = s->n_val_lanes;
  u64 key[MAXL], val[MAXL];
  for (u64 i = 0; i < n; i++) {
    for (int l = 0; l < nk; l++) key[l] = cols[l][i];
    for (int l = 0; l < nv; l++) val[l] = cols[nk + l][i];
    bld.push(key, val, w[i]);
  }
  *out = wrap(bld.done());
  return DBSP_OK;
}

int32_t orc_spine_new(orc_ctx* c, const dbsp_schema* s, orc_spine** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_new(WHAT, out, s));
  *out = new orc_spine(*s);
  return DBSP_OK;
}
int32_t orc_spine_insert(orc_ctx* c, orc_spine* s, const orc_batch* b) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_spine_insert(S(s), S(b)));
  s->s.insert(b->p);
  return DBSP_OK;
}
int32_t orc_spine_consolidate(orc_ctx* c, orc_spine* s, orc_batch** out) {
  NOT_NULL(c, "ctx");
  NOT_NULL(s, "spine");
  NOT_NULL(out, "out");
  *out = wrap(s->s.consolidate());
  return DBSP_OK;
}
int32_t orc_spine_truncate_keys_below(orc_ctx* c, orc_spine* s, const u64* key) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_truncate(WHAT, S(s), key, false));
  s->s.truncate(key);
  return DBSP_OK;
}
int32_t orc_spine_truncate_values_below(orc_ctx* c, orc_spine* s, const u64* val) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_truncate(WHAT, S(s), val, true));
  s->s.truncate_values(val);
  return DBSP_OK;
}
int32_t orc_spine_exert(orc_ctx* c, orc_spine* s, i64* effort) {
  NOT_NULL(c, "ctx");
  NOT_NULL(s, "spine");
  NOT_NULL(effort, "effort");
  s->s.exert(effort);
  return DBSP_OK;
}
int32_t orc_spine_len(const orc_spine* s, u64* n, uint32_t* nb) {
  NOT_NULL(s, "spine");
  if (n) *n = s->s.len();
  if (nb) *nb = (uint32_t)s->s.batches.size();
  return DBSP_OK;
}
int32_t orc_spine_free(orc_spine* s) { delete s; return DBSP_OK; }

// JoinTrace::eval with Time = () (operator/join.rs:732-863): the trace
// cursor is a CursorList over the spine's batches and map_times yields each
// batch's weight separately (:769-776), i.e. delta is joined with every batch
// and the outputs are consolidated by the Batcher (:845-858).
int32_t orc_join_delta_trace(orc_ctx* c, const orc_batch* delta, const orc_spine* tr, const dbsp_proj* proj,
                             int32_t delta_is_left, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_join(WHAT, out, S(delta), S(tr), delta_is_left, proj));
  Tuples t(proj->out_schema);
  for (auto& b : tr->s.batches) join_into(*delta->p, *b, *proj, !delta_is_left, t);
  *out = wrap(t.build());
  return DBSP_OK;
}

int32_t orc_join_batches(orc_ctx* c, const orc_batch* l, const orc_batch* r, const dbsp_proj* proj, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_join(WHAT, out, S(l), S(r), proj));
  Tuples t(proj->out_schema);
  join_into(*l->p, *r->p, *proj, false, t);
  *out = wrap(t.build());
  return DBSP_OK;
}

// SemiJoinStream::eval (operator/semijoin.rs:100-142).
int32_t orc_semijoin(orc_ctx* c, const orc_batch* pairs, const orc_batch* keys, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_semijoin(out, S(pairs), S(keys)));
  const Batch& P = *pairs->p;
  const Batch& Kb = *keys->p;
  // Out: ZSet<Key = (Pairs::Key, Pairs::Val)> (semijoin.rs:47): an OrdZSet over all lanes
  dbsp_schema os = P.s;
  os.n_key_lanes = (uint8_t)(P.s.n_key_lanes + P.s.n_val_lanes);
  os.n_val_lanes = 0;
  const int pnk = P.s.n_key_lanes, pnv = P.s.n_val_lanes;
  Builder bld(os);
  size_t i = 0, j = 0;
  u64 key[MAXL], val[MAXL];
  while (i < P.K.n && j < Kb.K.n) {
    int c = cmp_rows(P.K, i, Kb.K, j);
    if (c < 0) i++;
    else if (c > 0) j++;
    else {
      P.K.get(i, key);
      size_t lo, hi;
      P.vrange(i, lo, hi);
      for (size_t v = lo; v < hi; v++) {
        if (P.indexed()) { P.V.get(v, val); for (int l = 0; l < pnv; l++) key[pnk + l] = val[l]; }
        i64 w = (i64)((u64)P.w[v] * (u64)Kb.w[j]);
        if (w != 0) bld.push(key, val, w);
      }
      i++; j++;
    }
  }
  *out = wrap(bld.done());
  return DBSP_OK;
}

// AggregateIncremental::eval / eval_key (operator/aggregate/mod.rs:479-547,
// 600-684) producing (key, Option<out>) per delta key, then Upsert::eval
// (operator/upsert.rs:161-208): retract the key's current values in the
// output trace, insert the new one, consolidate per key.
int32_t orc_aggregate_delta(orc_ctx* c, const orc_batch* delta, const orc_spine* in_tr, const orc_spine* out_tr,
                            int32_t kind, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::valid_aggregate(out, S(delta), S(in_tr), S(out_tr), kind));
  const Batch& D = *delta->p;
  const dbsp_schema& os = out_tr->s.s;
  int nk = os.n_key_lanes, nov = os.n_val_lanes;
  Builder bld(os);
  std::vector<std::pair<KV, i64>> grp;
  u64 key[MAXL], key2[MAXL], newv[MAXL];
  size_t nkeys = D.K.n;
  for (size_t ki = 0; ki < nkeys; ki++) {
    D.K.get(ki, key);
    if (kind == DBSP_AGG_WCOUNT2) {
      // key = leading nk lanes of the (K.., which) row; visit each K once.
      if (ki > 0) { D.K.get(ki - 1, key2); if (cmp_tuples(D.s.lane_types, nk, key, key2) == 0) continue; }
    }
    bool has_new = false;
    if (kind == DBSP_AGG_MAX) {          // max.rs:36-55: walk back to the last value with weight != 0
      key_group(in_tr->s, key, grp);
      for (size_t g = grp.size(); g-- > 0;) if (grp[g].second != 0) { grp[g].first.b->V.get(grp[g].first.pos, newv); has_new = true; break; }
    } else if (kind == DBSP_AGG_MIN) {   // min.rs:38-57
      key_group(in_tr->s, key, grp);
      for (size_t g = 0; g < grp.size(); g++) if (grp[g].second != 0) { grp[g].first.b->V.get(grp[g].first.pos, newv); has_new = true; break; }
    } else if (kind == DBSP_AGG_FOLD_COUNT || kind == DBSP_AGG_FOLD_SUM) {   // fold.rs:76-96
      key_group(in_tr->s, key, grp);
      u64 acc = 0;
      for (auto& g : grp) if (g.second != 0) { has_new = true; acc += (kind == DBSP_AGG_FOLD_COUNT) ? 1 : g.first.b->V.c[0][g.first.pos]; }
      newv[0] = acc;
    } else if (kind == DBSP_AGG_WCOUNT) {   // aggregate/mod.rs:129-156
      key_group(in_tr->s, key, grp);
      i64 sum = 0;
      for (auto& g : grp) sum = (i64)((u64)sum + (u64)g.second);
      has_new = sum != 0; newv[0] = (u64)sum;
    } else if (kind == DBSP_AGG_WCOUNT2) {  // Avg is zero iff sum and count are both zero (average.rs:88-95)
      i64 sc[2] = {0, 0};
      for (int which = 0; which < 2; which++) {
        for (int l = 0; l < nk; l++) key2[l] = key[l];
        key2[nk] = (u64)which;
        key_group(in_tr->s, key2, grp);
        for (auto& g : grp) sc[which] = (i64)((u64)sc[which] + (u64)g.second);
      }
      has_new = sc[0] != 0 || sc[1] != 0; newv[0] = (u64)sc[0]; newv[1] = (u64)sc[1];
    } else return DBSP_ERR_INVALID;
    // Upsert::eval for this key.
    key_group(out_tr->s, key, grp);
    std::vector<std::pair<std::vector<u64>, i64>> upd;
    if (has_new) upd.push_back({std::vector<u64>(newv, newv + nov), 1});
    for (auto& g : grp) if (g.second != 0) {
      std::vector<u64> v(nov);
      g.first.b->V.get(g.first.pos, v.data());
      upd.push_back({v, (i64)((u64)0 - (u64)g.second)});
    }
    const uint8_t* vty = os.lane_types + nk;
    std::sort(upd.begin(), upd.end(), [&](auto& a, auto& b) { return cmp_tuples(vty, nov, a.first.data(), b.first.data()) < 0; });
    size_t i = 0;
    while (i < upd.size()) {
      size_t j = i; i64 sum = 0;
      while (j < upd.size() && cmp_tuples(vty, nov, upd[i].first.data(), upd[j].first.data()) == 0) { sum = (i64)((u64)sum + (u64)upd[j].second); j++; }
      if (sum != 0) bld.push(key, upd[i].first.data(), sum);
      i = j;
    }
  }
  *out = wrap(bld.done());
  return DBSP_OK;
}

// weigh (operator/aggregate/mod.rs:297-323).
int32_t orc_weigh(orc_ctx* c, const orc_batch* b, const dbsp_expr* f, int32_t mode, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_weigh(out, S(b), f, mode));
  const Batch& B = *b->p;
  dbsp_schema s = B.s;
  s.n_val_lanes = 0;
  if (mode == DBSP_WEIGH_AVG) { s.lane_types[s.n_key_lanes] = DBSP_U64; s.n_key_lanes++; }
  Builder bld(s);
  u64 key[MAXL], val[MAXL] = {0};
  for (size_t k = 0; k < B.K.n; k++) {
    B.K.get(k, key);
    size_t lo, hi;
    B.vrange(k, lo, hi);
    i64 agg = 0, cnt = 0;
    for (size_t v = lo; v < hi; v++) {
      if (B.indexed()) B.V.get(v, val);
      Env e{key, val, val};
      agg = (i64)((u64)agg + expr_val(*f, e) * (u64)B.w[v]);
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

// DistinctIncrementalTotal::eval (operator/distinct.rs:196-254).
int32_t orc_distinct_delta(orc_ctx* c, const orc_batch* delta, const orc_spine* integral, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_distinct_delta(out, S(delta), S(integral)));
  const Batch& D = *delta->p;
  Builder bld(D.s);
  std::vector<std::pair<KV, i64>> grp;
  u64 key[MAXL], val[MAXL];
  for (size_t k = 0; k < D.K.n; k++) {
    D.K.get(k, key);
    key_group(integral->s, key, grp);
    size_t lo, hi;
    D.vrange(k, lo, hi);
    for (size_t v = lo; v < hi; v++) {
      if (D.indexed()) D.V.get(v, val);
      i64 w = D.w[v], oldw = 0;
      for (auto& g : grp)
        if (!D.indexed() || cmp_row_tuple(g.first.b->V, g.first.pos, val) == 0) { oldw = g.second; break; }
      i64 neww = (i64)((u64)oldw + (u64)w);
      if (oldw <= 0) { if (neww > 0) bld.push(key, val, 1); }
      else if (neww <= 0) bld.push(key, val, -1);
    }
  }
  *out = wrap(bld.done());
  return DBSP_OK;
}

// IndexedZSet::distinct (algebra/zset/mod.rs:14-38).
int32_t orc_stream_distinct(orc_ctx* c, const orc_batch* b, orc_batch** out) {
  NOT_NULL(c, "ctx");
  NOT_NULL(out, "out");
  NOT_NULL(b, "batch");
  const Batch& B = *b->p;
  Builder bld(B.s);
  u64 key[MAXL], val[MAXL];
  for (size_t k = 0; k < B.K.n; k++) {
    B.K.get(k, key);
    size_t lo, hi;
    B.vrange(k, lo, hi);
    for (size_t v = lo; v < hi; v++) {
      if (B.indexed()) B.V.get(v, val);
      if (B.w[v] > 0) bld.push(key, val, 1);
    }
  }
  *out = wrap(bld.done());
  return DBSP_OK;
}

// Window::eval (operator/time_series/window.rs:144-222).
int32_t orc_window_delta(orc_ctx* c, const orc_spine* tr, const orc_batch* delta, int32_t has_prev, const u64* s0,
                         const u64* e0, const u64* s1, const u64* e1, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_window_delta(out, S(tr), S(delta), has_prev, s0, e0, s1, e1));
  const dbsp_schema& s = delta->p->s;
  int nk = s.n_key_lanes;
  Tuples t(s);
  u64 row[MAXL];
  auto lt = [&](const u64* a, const u64* b) { return cmp_tuples(s.lane_types, nk, a, b) < 0; };
  // emit keys of `b` in [from, min(until1, until2)) with weight * sign
  auto emit = [&](const Batch& b, const u64* from, const u64* until1, const u64* until2, int sign) {
    size_t k = seek_key(b, 0, from);
    for (; k < b.K.n; k++) {
      b.K.get(k, row);
      if (!lt(row, until1)) break;
      if (until2 && !lt(row, until2)) break;
      size_t lo, hi;
      b.vrange(k, lo, hi);
      for (size_t v = lo; v < hi; v++) {
        if (b.indexed()) b.V.get(v, row + nk);
        t.push(row, sign > 0 ? b.w[v] : (i64)((u64)0 - (u64)b.w[v]));
      }
    }
  };
  if (has_prev) {
    for (auto& b : tr->s.batches) {
      emit(*b, s0, s1, e0, -1);                       // region 1: slid out on the left
      if (lt(e1, e0)) emit(*b, e1, e0, nullptr, -1);  // window shrank on the right
      const u64* from = lt(e0, s1) ? s1 : e0;         // max(end0, start1)
      emit(*b, from, e1, nullptr, +1);                // region 3: slid in
    }
  }
  emit(*delta->p, s1, e1, nullptr, +1);
  *out = wrap(t.build());
  return DBSP_OK;
}

// Map/FlatMap::eval + from_tuples (operator/filter_map.rs:563-577,700-724).
int32_t orc_map_index(orc_ctx* c, const orc_batch* b, const dbsp_proj* proj, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_map_index(WHAT, out, S(b), proj));
  const Batch& B = *b->p;
  Tuples t(proj->out_schema);
  u64 key[MAXL], val[MAXL] = {0}, row[MAXL];
  for (size_t k = 0; k < B.K.n; k++) {
    B.K.get(k, key);
    size_t lo, hi;
    B.vrange(k, lo, hi);
    for (size_t v = lo; v < hi; v++) {
      if (B.indexed()) B.V.get(v, val);
      Env e{key, val, val};
      if (project(*proj, e, row)) t.push(row, B.w[v]);
    }
  }
  *out = wrap(t.build());
  return DBSP_OK;
}

// The shard hash.  The reference uses XXH3-64 (hash.rs:6-13); placement is
// unobservable after the union over workers (communication/shard.rs:38-51),
// so both the oracle and the CUDA path use this splitmix64 fold instead.
static inline u64 mix64(u64 x) {
  x += 0x9e3779b97f4a7c15ull;
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}
// shard_batch (operator/communication/shard.rs:165-199).
int32_t orc_shard_partition(orc_ctx* c, const orc_batch* b, uint32_t P, orc_batch** outs) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_shard_partition(S(b), outs, P));
  const Batch& B = *b->p;
  std::vector<Builder> blds;
  for (uint32_t p = 0; p < P; p++) blds.emplace_back(B.s);
  u64 key[MAXL], val[MAXL];
  for (size_t k = 0; k < B.K.n; k++) {
    B.K.get(k, key);
    u64 h = 0;
    for (int l = 0; l < B.K.nl; l++) h = mix64(h ^ key[l]);
    uint32_t p = (uint32_t)(h % P);
    size_t lo, hi;
    B.vrange(k, lo, hi);
    for (size_t v = lo; v < hi; v++) {
      if (B.indexed()) B.V.get(v, val);
      blds[p].push(key, val, B.w[v]);
    }
  }
  for (uint32_t p = 0; p < P; p++) outs[p] = wrap(blds[p].done());
  return DBSP_OK;
}

// Checkpoint / resume of a trace: the file format of dbsp_spine_save (include/dbsp_b200.h), so that a snapshot
// written by either library loads in the other.
static const char SPINE_MAGIC[8] = {'D', 'B', 'S', 'P', 'S', 'P', 'N', '1'};
static bool wr(FILE* f, const void* p, size_t n) { return n == 0 || fwrite(p, 1, n, f) == n; }
static bool rd(FILE* f, void* p, size_t n) { return n == 0 || fread(p, 1, n, f) == n; }
static bool save_flat(FILE* f, const BatchP& b) {
  u64 present = b ? 1 : 0, n = b ? b->len() : 0;
  if (!wr(f, &present, 8) || !wr(f, &n, 8)) return false;
  if (!n) return true;
  const Batch& B = *b;
  const int nk = B.s.n_key_lanes, nv = B.s.n_val_lanes;
  std::vector<u64> lane(n);
  for (int l = 0; l < nk; l++) {   // flat rows: every key repeated over its value range
    size_t o = 0;
    for (size_t k = 0; k < B.K.n; k++) { size_t lo, hi; B.vrange(k, lo, hi); for (size_t v = lo; v < hi; v++) lane[o++] = B.K.c[l][k]; }
    if (!wr(f, lane.data(), n * 8)) return false;
  }
  for (int l = 0; l < nv; l++) if (!wr(f, B.V.c[l].data(), n * 8)) return false;
  return wr(f, B.w.data(), n * 8);
}
// batch `which` (0 = a, 1 = b) of a layer of kind `kind`: checked before anything is allocated for it, and its rows
// checked — ordered, no duplicate rows, no zero weights — before they become a batch of the trace
static int32_t load_flat(FILE* f, u64 file_bytes, const dbsp_schema& sc, u64 kind, int which, BatchP* out) {
  u64 present = 0, n = 0;
  *out = nullptr;
  if (!rd(f, &present, 8) || !rd(f, &n, 8)) { g_err = "spine_load: truncated file (batch header)"; return DBSP_ERR_INVALID; }
  const int L = sc.n_key_lanes + sc.n_val_lanes;
  REFUSE(dv::valid_snapshot_batch(kind, which, present, n, L, file_bytes - (u64)ftell(f)));
  if (!present) return DBSP_OK;
  std::vector<std::vector<u64>> cols((size_t)L, std::vector<u64>(n));
  std::vector<i64> w(n);
  for (int l = 0; l < L; l++) if (!rd(f, cols[(size_t)l].data(), n * 8)) { g_err = "spine_load: truncated file (lane)"; return DBSP_ERR_INVALID; }
  if (!rd(f, w.data(), n * 8)) { g_err = "spine_load: truncated file (weights)"; return DBSP_ERR_INVALID; }
  u64 inv = 0, dup = 0, zero = 0, prev[MAXL], row[MAXL];
  Builder bld(sc);
  for (u64 i = 0; i < n; i++) {
    for (int l = 0; l < L; l++) row[l] = cols[(size_t)l][i];
    if (i) {
      const int c = cmp_tuples(sc.lane_types, L, prev, row);
      inv += c > 0;
      dup += c == 0;
    }
    zero += w[i] == 0;
    bld.push(row, row + sc.n_key_lanes, w[i]);
    memcpy(prev, row, sizeof(row));
  }
  if (inv || dup || zero) {
    g_err = "spine_load: rows of a batch are not consolidated (" + std::to_string(inv) + " out of order, " + std::to_string(dup) +
            " duplicates, " + std::to_string(zero) + " zero weights)";
    return DBSP_ERR_INVALID;
  }
  *out = bld.done();
  return DBSP_OK;
}
int32_t orc_spine_save(orc_ctx* c, const orc_spine* sp, const char* path) {
  NOT_NULL(c, "ctx");
  NOT_NULL(sp, "spine");
  NOT_NULL(path, "path");
  const Spine& s = sp->s;
  FILE* f = fopen(path, "wb");
  if (!f) { g_err = "spine_save: cannot open file"; return DBSP_ERR_INVALID; }
  u64 hdr[4] = {s.has_bound ? 1ull : 0ull, s.has_vbound ? 1ull : 0ull, (u64)s.effort, (u64)s.merging.size()};
  bool ok = wr(f, SPINE_MAGIC, 8) && wr(f, &s.s, sizeof(dbsp_schema)) && wr(f, hdr, sizeof(hdr)) && wr(f, s.bound, 8 * MAXL) && wr(f, s.vbound, 8 * MAXL);
  for (size_t i = 0; ok && i < s.merging.size(); i++) {
    const Spine::Layer& l = s.merging[i];
    // a merge in progress is written as its two inputs plus the fuel still owed (inputs not yet consumed)
    u64 owed = 0;
    if (l.kind == Spine::Layer::IN_PROGRESS) owed = (u64)(l.a->len() + l.b->len());
    u64 lh[2] = {(u64)l.kind, owed};
    ok = wr(f, lh, sizeof(lh)) && save_flat(f, l.a) && save_flat(f, l.kind == Spine::Layer::IN_PROGRESS ? l.b : nullptr);
  }
  ok = (fclose(f) == 0) && ok;
  if (!ok) { g_err = "spine_save: write failed"; return DBSP_ERR_INVALID; }
  return DBSP_OK;
}
static int32_t load_spine(FILE* f, std::unique_ptr<orc_spine>& sp) {
  u64 file_bytes = 0;
  if (fseek(f, 0, SEEK_END) == 0) { file_bytes = (u64)ftell(f); rewind(f); }
  char magic[8];
  dbsp_schema sc;
  u64 hdr[4], bound[MAXL], vbound[MAXL];
  if (!rd(f, magic, 8) || memcmp(magic, SPINE_MAGIC, 8) != 0) { g_err = "spine_load: not a spine snapshot (magic)"; return DBSP_ERR_INVALID; }
  if (!rd(f, &sc, sizeof(sc)) || !rd(f, hdr, sizeof(hdr)) || !rd(f, bound, 8 * MAXL) || !rd(f, vbound, 8 * MAXL)) {
    g_err = "spine_load: truncated file (header)";
    return DBSP_ERR_INVALID;
  }
  REFUSE(dv::valid_snapshot_header(sc, hdr));
  sp.reset(new orc_spine(sc));
  Spine& s = sp->s;
  memcpy(s.bound, bound, sizeof(bound));
  memcpy(s.vbound, vbound, sizeof(vbound));
  s.has_bound = hdr[0] != 0;
  s.has_vbound = hdr[1] != 0;
  s.effort = hdr[2] ? (size_t)hdr[2] : 1;
  for (u64 i = 0; i < hdr[3]; i++) {
    u64 lh[2];
    if (!rd(f, lh, sizeof(lh))) { g_err = "spine_load: truncated file (layer header)"; return DBSP_ERR_INVALID; }
    REFUSE(dv::valid_snapshot_kind(lh[0]));
    Spine::Layer l;
    int32_t rc = load_flat(f, file_bytes, sc, lh[0], 0, &l.a);
    if (rc == DBSP_OK) rc = load_flat(f, file_bytes, sc, lh[0], 1, &l.b);
    if (rc != DBSP_OK) return rc;
    REFUSE(dv::valid_snapshot_remaining(lh[1], l.a ? l.a->len() : 0, l.b ? l.b->len() : 0));
    l.kind = (Spine::Layer::Kind)lh[0];
    if (l.kind == Spine::Layer::IN_PROGRESS) l.m = std::make_shared<Merger>(l.a, l.b);   // the merge restarts; its inputs and its place in the schedule are kept
    s.merging.push_back(l);
  }
  if ((u64)ftell(f) != file_bytes) { g_err = "spine_load: " + std::to_string(file_bytes - (u64)ftell(f)) + " trailing bytes after the last layer"; return DBSP_ERR_INVALID; }
  return DBSP_OK;
}
int32_t orc_spine_load(orc_ctx* c, const char* path, orc_spine** out) {
  NOT_NULL(c, "ctx");
  NOT_NULL(path, "path");
  NOT_NULL(out, "out");
  FILE* f = fopen(path, "rb");
  if (!f) { g_err = "spine_load: cannot open file"; return DBSP_ERR_INVALID; }
  std::unique_ptr<orc_spine> sp;   // a refused file leaves nothing behind
  const int32_t rc = load_spine(f, sp);
  fclose(f);
  if (rc != DBSP_OK) return rc;
  sp->s.refresh();
  *out = sp.release();
  return DBSP_OK;
}

// Communication entry points of the ABI.  The oracle is one worker: identity for world == 1 (shard.rs:111-114);
// the multi-worker CPU runs use the in-process exchange of oracle/nexmark_workers.cpp / thread_workers.py.
int32_t orc_comm_create(orc_ctx* c, int32_t rank, int32_t world, u64, uint8_t* blob) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_comm_create(rank, world, blob));
  if (world != 1 || rank != 0) { g_err = "oracle: single worker only"; return DBSP_ERR_UNSUPPORTED; }
  if (blob) memset(blob, 0, DBSP_COMM_BLOB_BYTES);
  return DBSP_OK;
}
int32_t orc_comm_connect(orc_ctx* c, const uint8_t* blobs) {
  NOT_NULL(c, "ctx");
  NOT_NULL(blobs, "blobs");
  return DBSP_OK;
}
int32_t orc_comm_destroy(orc_ctx* c) { NOT_NULL(c, "ctx"); return DBSP_OK; }
int32_t orc_comm_info(orc_ctx* c, int32_t* rank, int32_t* world, u64* bytes) {
  NOT_NULL(c, "ctx");
  if (rank) *rank = 0;
  if (world) *world = 1;
  if (bytes) *bytes = 0;
  return DBSP_OK;
}
int32_t orc_shard(orc_ctx* c, const orc_batch* b, orc_batch** out) {
  NOT_NULL(c, "ctx");
  NOT_NULL(out, "out");
  NOT_NULL(b, "batch");
  *out = wrap(b->p);
  return DBSP_OK;
}
int32_t orc_shard2(orc_ctx* c, const orc_batch* a, const orc_batch* b, orc_batch** oa, orc_batch** ob) {
  NOT_NULL(c, "ctx");
  NOT_NULL(oa, "out_a");
  NOT_NULL(ob, "out_b");
  NOT_NULL(a, "a");
  NOT_NULL(b, "b");
  *oa = wrap(a->p);
  *ob = wrap(b->p);
  return DBSP_OK;
}
int32_t orc_gather(orc_ctx* c, const orc_batch* b, int32_t root, orc_batch** out) {
  NOT_NULL(c, "ctx");
  REFUSE(dv::check_gather(out, S(b), root, 1));
  *out = wrap(b->p);
  return DBSP_OK;
}
int32_t orc_allreduce_max_u64(orc_ctx* c, u64* x) { NOT_NULL(c, "ctx"); NOT_NULL(x, "x"); return DBSP_OK; }

}  // extern "C"
