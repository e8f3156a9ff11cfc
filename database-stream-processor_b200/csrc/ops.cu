// ops.cu — operator kernels: projection/filter, delta-vs-trace probes (join,
// aggregate, distinct), window ranges, shard partition.  Each host entry
// cites the reference `eval` it replaces (paths under crates/dbsp/src/).
#include <cub/device/device_scan.cuh>

#include "ops.cuh"
#include "validate.h"

namespace {

constexpr int TB = 256;

// up to MAX_REFS spine batches passed to a kernel by value
struct BatchRef {
  Cols c;
  const i64* w;
  u64 n;
};
constexpr int MAX_REFS = 16;
struct BatchRefs {
  BatchRef b[MAX_REFS];
  int nb;
};

// ---------------- declarative row expressions on the device ------------------
struct Env {
  const u64* key;
  const u64* lv;
  const u64* rv;
  __device__ __forceinline__ u64 k(int i) const { return key[i]; }
  __device__ __forceinline__ u64 l(int i) const { return lv[i]; }
  __device__ __forceinline__ u64 r(int i) const { return rv[i]; }
};
// one row of a column table / batch, read in place: only the lanes the closure names are ever loaded
struct ColEnv {
  const Cols& c;
  int nk;
  u64 row;
  __device__ __forceinline__ u64 k(int i) const { return c.c[i][row]; }
  __device__ __forceinline__ u64 l(int i) const { return c.c[nk + i][row]; }
  __device__ __forceinline__ u64 r(int i) const { return c.c[nk + i][row]; }
};
// one run of a fan-out (dbsp_*_fanout): input row `row` of a column table, generating output j (DBSP_SRC_FANOUT)
struct FanEnv {
  const Cols& c;
  int nk;
  u64 row;
  u64 j;
  __device__ __forceinline__ u64 k(int i) const { return c.c[i][row]; }
  __device__ __forceinline__ u64 l(int i) const { return c.c[nk + i][row]; }
  __device__ __forceinline__ u64 r(int i) const { return c.c[nk + i][row]; }
};
// one step of a Fold (dbsp_fold): row `row` of a gathered key group, the accumulator and the row's summed weight
// (DBSP_SRC_ACC / DBSP_SRC_WEIGHT); the output program runs in it too, reading only the key and the accumulator
struct FoldEnv {
  const Cols& c;
  int nk;
  u64 row;
  const u64* acc;
  i64 w;
  __device__ __forceinline__ u64 k(int i) const { return c.c[i][row]; }
  __device__ __forceinline__ u64 l(int i) const { return c.c[nk + i][row]; }
  __device__ __forceinline__ u64 r(int i) const { return c.c[nk + i][row]; }
};
template <class E>
__device__ __forceinline__ u64 src_val(const dbsp_src& s, const E& e) {
  switch (s.kind) {
    case DBSP_SRC_KEY: return e.k(s.idx);
    case DBSP_SRC_LVAL: return e.l(s.idx);
    case DBSP_SRC_RVAL: return e.r(s.idx);
    default: return (u64)s.cst;
  }
}
template <class E>
__device__ __forceinline__ u64 expr_val(const dbsp_expr& x, const E& e) {
  u64 a = src_val(x.a, e);
  switch (x.op) {
    case DBSP_OP_COPY: return a;
    case DBSP_OP_NEG: return (u64)0 - a;
    case DBSP_OP_ADD: return a + src_val(x.b, e);
    case DBSP_OP_SUB: return a - src_val(x.b, e);
    case DBSP_OP_MUL: return a * src_val(x.b, e);
    case DBSP_OP_DIV: {   // i64::wrapping_div, x / 0 = 0: MIN / -1 wraps to MIN instead of trapping
      i64 d = (i64)src_val(x.b, e);
      if (d == 0) return 0;
      if (d == -1) return (u64)0 - a;
      return (u64)((i64)a / d);
    }
  }
  return a;
}
template <class E>
__device__ __forceinline__ bool pred_ok(const dbsp_pred& p, const E& e) {
  u64 a = src_val(p.a, e), b = src_val(p.b, e);
  if (p.cmp == DBSP_CMP_IN) return a < 64 && ((b >> a) & 1);
  int c = p.is_signed ? (((i64)a < (i64)b) ? -1 : ((i64)a > (i64)b)) : ((a < b) ? -1 : (a > b));
  switch (p.cmp) {
    case DBSP_CMP_EQ: return c == 0;
    case DBSP_CMP_NE: return c != 0;
    case DBSP_CMP_LT: return c < 0;
    case DBSP_CMP_LE: return c <= 0;
    case DBSP_CMP_GT: return c > 0;
    case DBSP_CMP_GE: return c >= 0;
  }
  return false;
}
// evaluates the output row unconditionally (a filtered row keeps its place in
// an ordered output with weight 0) and returns whether the predicates hold
__device__ __forceinline__ bool project(const dbsp_proj& p, const Env& e, u64* row) {
  bool ok = true;
  for (int i = 0; i < p.n_pred; i++) ok = ok && pred_ok(p.pred[i], e);
  int nl = p.out_schema.n_key_lanes + p.out_schema.n_val_lanes;
  for (int l = 0; l < nl; l++) row[l] = expr_val(p.out[l], e);
  return ok;
}

// Row function (dbsp_rowfn): the postfix program leaves the output lanes and the keep flag in st[0..L].  The program
// is a kernel parameter, the same for every thread, so the dispatch is warp-uniform; the stack is a local array
// indexed by the (uniform) depth.  validate.h has checked the depths and sources, and every operation is total.
template <class E>
__device__ __forceinline__ void run_rowfn(const dbsp_rowfn& f, const E& e, u64* st) {
  int sp = 0;
#pragma unroll 1
  for (int pc = 0; pc < f.n_insn; pc++) {
    const dbsp_insn& in = f.code[pc];
    const int op = in.op;
    if (op == DBSP_FN_PUSH) {
      u64 v;
      switch (in.kind) {
        case DBSP_SRC_KEY: v = e.k(in.idx); break;
        case DBSP_SRC_LVAL: v = e.l(in.idx); break;
        case DBSP_SRC_RVAL: v = e.r(in.idx); break;
        default:
          if constexpr (std::is_same<E, FanEnv>::value) {   // only a fan-out's environment has a j
            if (in.kind == DBSP_SRC_FANOUT) { v = e.j; break; }
          }
          if constexpr (std::is_same<E, FoldEnv>::value) {   // only a fold's environment has acc and a weight
            if (in.kind == DBSP_SRC_ACC) { v = e.acc[in.idx]; break; }
            if (in.kind == DBSP_SRC_WEIGHT) { v = (u64)e.w; break; }
          }
          v = (u64)in.cst;
      }
      st[sp++] = v;
      continue;
    }
    if (op <= DBSP_FN_LNOT) {
      const u64 a = st[sp - 1];
      u64 r;
      switch (op) {
        case DBSP_FN_NEG: r = (u64)0 - a; break;
        case DBSP_FN_ABS: r = (i64)a < 0 ? (u64)0 - a : a; break;
        case DBSP_FN_BNOT: r = ~a; break;
        default: r = a == 0;
      }
      st[sp - 1] = r;
      continue;
    }
    if (op == DBSP_FN_SELECT) {
      st[sp - 3] = st[sp - 3] ? st[sp - 2] : st[sp - 1];
      sp -= 2;
      continue;
    }
    const u64 b = st[--sp], a = st[sp - 1];
    const i64 sa = (i64)a, sb = (i64)b;
    u64 r;
    switch (op) {
      case DBSP_FN_ADD: r = a + b; break;
      case DBSP_FN_SUB: r = a - b; break;
      case DBSP_FN_MUL: r = a * b; break;
      case DBSP_FN_DIV: r = sb == 0 ? 0 : sb == -1 ? (u64)0 - a : (u64)(sa / sb); break;   // no MIN / -1 trap
      case DBSP_FN_REM: r = (sb == 0 || sb == -1) ? 0 : (u64)(sa % sb); break;
      case DBSP_FN_DIVU: r = b == 0 ? 0 : a / b; break;
      case DBSP_FN_REMU: r = b == 0 ? 0 : a % b; break;
      case DBSP_FN_MIN: r = sa < sb ? a : b; break;
      case DBSP_FN_MAX: r = sa > sb ? a : b; break;
      case DBSP_FN_MINU: r = a < b ? a : b; break;
      case DBSP_FN_MAXU: r = a > b ? a : b; break;
      case DBSP_FN_AND: r = a & b; break;
      case DBSP_FN_OR: r = a | b; break;
      case DBSP_FN_XOR: r = a ^ b; break;
      case DBSP_FN_SHL: r = a << (b & 63); break;
      case DBSP_FN_SHR: r = a >> (b & 63); break;
      case DBSP_FN_SAR: r = (u64)(sa >> (b & 63)); break;
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
      default: r = a < 64 && ((b >> a) & 1);   // DBSP_FN_IN
    }
    st[sp - 1] = r;
  }
}

// The closure forms the kernels that evaluate closures are instantiated on (dbsp_proj / dbsp_rowfn; for weigh
// dbsp_expr / dbsp_rowfn).  fn_keep: the row passes the filter; fn_emit: put(l, output lane l) for l < nl;
// project: both, into row[]; fn_factor: the weigh factor (0 for a filtered row) and whether the row counts.
template <class E>
__device__ __forceinline__ bool fn_keep(const dbsp_proj& p, const E& e) {
  bool ok = true;
  for (int q = 0; q < p.n_pred; q++) ok = ok && pred_ok(p.pred[q], e);
  return ok;
}
template <class E, class Put>
__device__ __forceinline__ void fn_emit(const dbsp_proj& p, const E& e, int nl, Put put) {
  for (int l = 0; l < nl; l++) put(l, expr_val(p.out[l], e));
}
template <class E>
__device__ __forceinline__ bool fn_keep(const dbsp_rowfn& f, const E& e) {
  u64 st[DBSP_MAX_STACK];
  run_rowfn(f, e, st);
  return st[f.out_schema.n_key_lanes + f.out_schema.n_val_lanes] != 0;
}
template <class E, class Put>
__device__ __forceinline__ void fn_emit(const dbsp_rowfn& f, const E& e, int nl, Put put) {
  u64 st[DBSP_MAX_STACK];
  run_rowfn(f, e, st);
  for (int l = 0; l < nl; l++) put(l, st[l]);
}
__device__ __forceinline__ bool project(const dbsp_rowfn& f, const Env& e, u64* row) {
  u64 st[DBSP_MAX_STACK];
  run_rowfn(f, e, st);
  const int nl = f.out_schema.n_key_lanes + f.out_schema.n_val_lanes;
  for (int l = 0; l < nl; l++) row[l] = st[l];
  return st[nl] != 0;
}
__device__ __forceinline__ bool fn_factor(const dbsp_expr& fx, const Env& e, u64* fv) {
  *fv = expr_val(fx, e);
  return true;
}
__device__ __forceinline__ bool fn_factor(const dbsp_rowfn& f, const Env& e, u64* fv) {
  u64 st[DBSP_MAX_STACK];
  run_rowfn(f, e, st);
  const bool keep = st[1] != 0;   // one output lane
  *fv = keep ? st[0] : 0;
  return keep;
}

// The virtual rows of k_project_rows.  For dbsp_proj / dbsp_rowfn virtual row v is input row v; for a fan-out
// (RowFnFanout) it is v = i * n_out + j, so the outputs keep the input order with j ascending inside each input row,
// and v < 2^32 (capi.cu refuses larger fan-outs from the sizes).
template <class F>
__device__ __forceinline__ u64 in_row(const F&, u64 v) { return v; }
__device__ __forceinline__ u64 in_row(const RowFnFanout& f, u64 v) { return (u32)v / f.n_out; }
template <class F>
__device__ __forceinline__ ColEnv row_env(const F&, const Cols& in, int nk, u64 v) { return ColEnv{in, nk, v}; }
__device__ __forceinline__ FanEnv row_env(const RowFnFanout& f, const Cols& in, int nk, u64 v) {
  const u32 i = (u32)v / f.n_out;
  return FanEnv{in, nk, i, (u32)v - i * f.n_out};
}

// flat_map_index over a raw table (filter_map.rs:700-724) / map_index over a
// batch, in one pass and order preserving: a CTA evaluates the predicates of its PROJ_ROWS rows, a decoupled
// look-back over the CTA totals gives it its output base, and the survivors' output rows are evaluated and written
// in input order — so inputs that are already ordered on the output key (id-ordered event tables, monotone
// projections) reach the sort-free path of consolidate_rows.  The surviving-row count stays on the device
// (*d_m): the census of consolidate_rows returns it.  identity != 0 (no predicates): output slot = input row.
constexpr int PROJ_IT = 4;
constexpr int PROJ_ROWS = TB * PROJ_IT;
template <class F>
__global__ void __launch_bounds__(TB)
k_project_rows(Cols in, int nk_in, const i64* w, u64 n, F proj, int identity, u32 ntiles, u32* ticket,
               u64* status, MCols out, i64* out_w, u32* d_m) {
  static_assert(PROJ_IT * (TB / 32) == 32, "one warp scans the per-(round, warp) counts");
  __shared__ u32 s_tile;
  __shared__ u32 s_cnt[32], s_off[32];
  __shared__ u64 s_base;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int nl = proj.out_schema.n_key_lanes + proj.out_schema.n_val_lanes;
  if (identity) {
    const u64 base = (u64)blockIdx.x * PROJ_ROWS;
    for (int it = 0; it < PROJ_IT; it++) {
      const u64 i = base + (u64)it * TB + tid;
      if (i < n) {
        const auto e = row_env(proj, in, nk_in, i);
        fn_emit(proj, e, nl, [&](int l, u64 v) { out.c[l][i] = v; });
        out_w[i] = w ? w[in_row(proj, i)] : 1;
      }
    }
    return;
  }
  if (tid == 0) s_tile = atomicAdd(ticket, 1u);
  __syncthreads();
  const u32 t = s_tile;
  const u64 base_row = (u64)t * PROJ_ROWS;
  unsigned okbits = 0, rk = 0;   // rk: 8 bits per round = number of surviving rows before this lane in its warp
  for (int it = 0; it < PROJ_IT; it++) {
    const u64 i = base_row + (u64)it * TB + tid;
    bool ok = false;
    if (i < n) {
      const auto e = row_env(proj, in, nk_in, i);
      ok = fn_keep(proj, e);
    }
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) s_cnt[it * (TB / 32) + wid] = __popc(m);
    if (ok) {
      okbits |= 1u << it;
      rk |= (unsigned)__popc(m & ((1u << lane) - 1)) << (8 * it);
    }
  }
  __syncthreads();
  if (wid == 0) {
    const u32 c = s_cnt[lane];
    u32 incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const u32 v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    const u32 total = __shfl_sync(0xffffffffu, incl, 31);
    s_off[lane] = incl - c;
    const u64 base = lb_exclusive_prefix(status, t, (u64)total);
    if (lane == 0) {
      s_base = base;
      if (t == ntiles - 1) *d_m = (u32)(base + total);
    }
  }
  __syncthreads();
  const u64 base = s_base;
  for (int it = 0; it < PROJ_IT; it++) {
    if (!((okbits >> it) & 1)) continue;
    const u64 i = base_row + (u64)it * TB + tid;
    const u64 pos = base + s_off[it * (TB / 32) + wid] + ((rk >> (8 * it)) & 0xffu);
    const auto e = row_env(proj, in, nk_in, i);
    fn_emit(proj, e, nl, [&](int l, u64 v) { out.c[l][pos] = v; });
    out_w[pos] = w ? w[in_row(proj, i)] : 1;
  }
}

// ---------------- delta x trace probes -----------------------------------------
// Warp range search: the rows of 32 consecutive distinct sorted query keys (one per lane) in each batch of a launch.
// Most probes touch few batches (ids grow from step to step, so a step's keys sit in the newest batches or above
// all of them), and a thread walking every batch alone runs ~log2(n) dependent loads per batch.  Instead:
// - bounds test: the first and last key of every batch sit in shared memory; a batch that the warp's key span
//   [q_min, q_max] misses is skipped by the whole warp without a global load;
// - shared window: the warp narrows [lower_bound(q_min), upper_bound(q_max)) together, 32 pivots per round and a
//   ballot per bound, so a window shrinks ~32x per round of independent loads;
// - per lane: lower bound by bisection inside that window, upper bound by galloping (the `seek_key` of
//   cursor/mod.rs + advance.rs:25-72) capped at the window's end.
// The search is exact: a key with rows in a batch gets its lower bound and count there.  A key without rows gets
// hi == lo and an unspecified lo: no caller reads lo for an empty range.
// The shared window stops narrowing at this width: a round's pivots are then spread over every warp of the launch
// and miss the cache, so a round costs more than the bisection steps it saves the lanes (random keys, 10 M-row
// batches, measured on an H100).
constexpr u64 WIN_MIN = 1024;
struct BatchBounds {
  u64 first[MAX_REFS][MAXL], last[MAX_REFS][MAXL];   // flipped like the queries; unset for an empty batch
  u64 q[TB / 32][2][MAXL];                            // per warp: its smallest and its largest query key
};
// every thread of the block calls it (it ends in a barrier)
__device__ __forceinline__ void load_bounds(BatchBounds& s, const BatchRefs& tr, int nk, const Flips& f) {
  for (int i = threadIdx.x; i < tr.nb * 2 * nk; i += blockDim.x) {
    const int b = i / (2 * nk), l = i % nk;
    const bool last = i % (2 * nk) >= nk;
    const u64 n = tr.b[b].n;
    if (n) (last ? s.last : s.first)[b][l] = tr.b[b].c.c[l][last ? n - 1 : 0] ^ f.f[l];
  }
  __syncthreads();
}
__device__ __forceinline__ int cmp_keys(const u64* a, const u64* b, int nk) {
  for (int l = 0; l < nk; l++)
    if (a[l] != b[l]) return a[l] < b[l] ? -1 : 1;
  return 0;
}
// Lanes [0, nact) hold the warp's keys in ascending order, q of an idle lane is not read.  Publishes the warp's key
// span for warp_key_range; every lane calls it.
__device__ __forceinline__ void warp_key_span(BatchBounds& s, const u64* q, int nact, int nk) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  __syncwarp();   // the previous span's readers are done
  if (lane == 0) for (int l = 0; l < nk; l++) s.q[wid][0][l] = q[l];
  if (lane == nact - 1) for (int l = 0; l < nk; l++) s.q[wid][1][l] = q[l];
  __syncwarp();
}
// One round of a 32-ary search for the first row of [a, b) whose predicate holds (b if none): lane j tested the
// pivot a + j*m/32, m = b - a, and `bal` is the ballot.  The answer stays in [a, b].
__device__ __forceinline__ void narrow(u64& a, u64& b, u64 m, unsigned bal) {
  if (m == 0) return;
  if (!bal) { a += (31 * m >> 5) + 1; return; }
  const u64 j = (u64)(__ffs(bal) - 1);   // pivot j - 1 < pivot j: equal pivots give equal predicates
  b = a + (j * m >> 5);
  if (j) a += ((j - 1) * m >> 5) + 1;
}
// [lo, hi) of this lane's key q (flipped) in batch b of s; `active`: the lane holds a key.  Every lane of the warp
// calls it with the same batch.
__device__ __forceinline__ void warp_key_range(const BatchBounds& s, const BatchRefs& tr, int b, const u64* q,
                                               bool active, int nk, const Flips& f, u64& lo, u64& hi) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const u64* qmin = s.q[wid][0];
  const u64* qmax = s.q[wid][1];
  const u64 nt = tr.b[b].n;
  lo = hi = 0;
  if (nt == 0 || cmp_keys(qmax, s.first[b], nk) < 0 || cmp_keys(qmin, s.last[b], nk) > 0) return;
  const Cols& T = tr.b[b].c;
  u64 a0 = 0, b0 = nt, a1 = 0, b1 = nt;   // lower_bound(qmin) in [a0, b0], upper_bound(qmax) in [a1, b1]
  while (b0 - a0 > WIN_MIN || b1 - a1 > WIN_MIN) {
    const u64 m0 = b0 - a0, m1 = b1 - a1;
    const bool g0 = m0 && cmp_row_q(T, a0 + ((u64)lane * m0 >> 5), qmin, nk, f) >= 0;
    const bool g1 = m1 && cmp_row_q(T, a1 + ((u64)lane * m1 >> 5), qmax, nk, f) > 0;
    narrow(a0, b0, m0, __ballot_sync(0xffffffffu, g0));
    narrow(a1, b1, m1, __ballot_sync(0xffffffffu, g1));
  }
  if (!active) return;
  const u64 top = b1;   // every key of the warp lies in rows [a0, b1)
  lo = lower_bound_q(T, a0, top, q, nk, f);
  hi = lo;
  u64 step = 1;
  while (hi + step <= top && cmp_row_q(T, hi + step - 1, q, nk, f) == 0) { hi += step; step <<= 1; }
  hi = upper_bound_q(T, hi, hi + step <= top ? hi + step : top, q, nk, f);
}

// Per *distinct* delta key (delta rows are sorted, so a key's rows are one segment [kstart[k], kstart[k+1])) and
// per trace batch: the range of trace rows carrying that key.  One search per key instead of one per row; a warp
// per 32 keys; all spine batches in one launch.
__global__ void k_probe_keys(Cols D, const u64* kstart, const u32* d_nkeys, BatchRefs tr, int nk, Flips f, u32* lo_out, u32* cnt_out,
             u32* ktot) {
  __shared__ BatchBounds s;
  load_bounds(s, tr, nk, f);
  const int lane = threadIdx.x & 31;
  const u64 nkeys = (u64)*d_nkeys;   // the exact key count lives on the device; the grid is a fixed-size grid-stride loop
  for (u64 base = (u64)blockIdx.x * TB + (threadIdx.x & ~31); base < nkeys; base += (u64)gridDim.x * TB) {
    const u64 k = base + lane;
    const bool active = k < nkeys;
    u64 q[MAXL];
    if (active) {
      const u64 row = kstart[k];
      for (int l = 0; l < nk; l++) q[l] = D.c[l][row] ^ f.f[l];
    }
    warp_key_span(s, q, (int)min(nkeys - base, (u64)32), nk);
    u64 tot = 0;
    for (int b = 0; b < tr.nb; b++) {
      u64 lo, hi;
      warp_key_range(s, tr, b, q, active, nk, f, lo, hi);
      if (active) {
        lo_out[k * tr.nb + b] = (u32)lo;
        cnt_out[k * tr.nb + b] = (u32)(hi - lo);
      }
      tot += hi - lo;
    }
    if (active) ktot[k] = tot > 0xffffffffull ? 0xffffffffu : (u32)tot;   // saturate: the 64-bit total below then trips the guard
  }
}

// Key segments of a sorted batch in one pass: a row is a head when it differs from its predecessor over the
// first nk lanes.  Each thread owns SEG_IPT consecutive rows; block scan of the head counts + decoupled look-back
// over the tiles give every head its key index: kstart[key] = row, ki[row] = key of the row, kstart[nkeys] = n
// and *d_nkeys = nkeys (the key count never leaves the device).
constexpr int SEG_IPT = 4, SEG_TILE = TB * SEG_IPT;
__global__ void __launch_bounds__(TB)
k_key_segments(Cols C, u64 n, int nk, u32 ntiles, u32* ticket, u64* status, u64* kstart, u32* ki, u32* d_nkeys) {
  __shared__ u32 s_tile, s_warp[TB / 32];
  __shared__ u64 s_base;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) s_tile = atomicAdd(ticket, 1u);
  __syncthreads();
  const u32 t = s_tile;
  const u64 i0 = (u64)t * SEG_TILE + (u64)tid * SEG_IPT;
  unsigned heads = 0;
#pragma unroll
  for (int k = 0; k < SEG_IPT; k++) {
    const u64 i = i0 + k;
    if (i < n) {
      bool head = i == 0;
      if (!head)
        for (int l = 0; l < nk; l++)
          if (C.c[l][i] != C.c[l][i - 1]) { head = true; break; }
      heads |= (head ? 1u : 0u) << k;
    }
  }
  const u32 cnt = __popc(heads);
  u32 incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const u32 v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) s_warp[wid] = incl;
  __syncthreads();
  u32 woff = 0, tile_total = 0;
#pragma unroll
  for (int k = 0; k < TB / 32; k++) {
    const u32 v = s_warp[k];
    if (k < wid) woff += v;
    tile_total += v;
  }
  if (wid == 0) {
    const u64 base = lb_exclusive_prefix(status, t, (u64)tile_total);
    if (lane == 0) {
      s_base = base;
      if (t == ntiles - 1) {
        *d_nkeys = (u32)(base + tile_total);
        kstart[base + tile_total] = n;
      }
    }
  }
  __syncthreads();
  u32 run = (u32)s_base + woff + incl - cnt;   // heads before this thread's first row
#pragma unroll
  for (int k = 0; k < SEG_IPT; k++) {
    const u64 i = i0 + k;
    if (i < n) {
      if ((heads >> k) & 1) { kstart[run] = i; run++; }
      ki[i] = run - 1;
    }
  }
}

// matches of every delta row = matches of its key, and their exclusive running sum (the output slot of the row's
// first match) in the same pass: ex[i] for i < nd, ex[nd] = total.  The total is carried in 64 bits through the
// look-back (a skewed join can exceed 2^32 matches; the 32-bit ex[] wraps then, and the host rejects the step on
// the exact total, which the last tile publishes to the host mailbox).
__global__ void __launch_bounds__(TB)
k_row_counts_scan(const u32* __restrict__ ki, const u32* __restrict__ ktot, u64 nd, u32 ntiles, u32* ticket, u64* status,
                  u32* ex, Mail mail) {
  __shared__ u32 s_tile;
  __shared__ u64 s_warp[TB / 32];
  __shared__ u64 s_base;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) s_tile = atomicAdd(ticket, 1u);
  __syncthreads();
  const u32 t = s_tile;
  const u64 i0 = (u64)t * SEG_TILE + (u64)tid * SEG_IPT;
  u32 c[SEG_IPT];
  u64 sum = 0;
#pragma unroll
  for (int k = 0; k < SEG_IPT; k++) {
    c[k] = (i0 + k < nd) ? ktot[ki[i0 + k]] : 0u;
    sum += c[k];
  }
  u64 incl = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const u64 v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) s_warp[wid] = incl;
  __syncthreads();
  u64 woff = 0, tile_total = 0;
#pragma unroll
  for (int k = 0; k < TB / 32; k++) {
    const u64 v = s_warp[k];
    if (k < wid) woff += v;
    tile_total += v;
  }
  if (wid == 0) {
    const u64 base = lb_exclusive_prefix(status, t, tile_total);
    if (lane == 0) {
      s_base = base;
      if (t == ntiles - 1) {
        const u64 tot = base + tile_total;
        ex[nd] = (u32)tot;
        mail_publish(mail, &tot, 1);
      }
    }
  }
  __syncthreads();
  u64 run = s_base + woff + incl - sum;
#pragma unroll
  for (int k = 0; k < SEG_IPT; k++) {
    if (i0 + k < nd) ex[i0 + k] = (u32)run;
    run += c[k];
  }
}

// Expand the matches: output slot o -> (delta row i, batch b, trace row).  Slots
// are ordered by (delta row, batch, trace row): for a monotone join_func and keys
// that live in a single batch that is already the output order, so consolidation
// needs no sort.  proj_mode 1: join_func(k, v1, v2) with filter
// (join.rs:751-787), weight w1*w2, rejected rows keep their slot with weight 0;
// proj_mode 0: copy the trace row (gather of a key group).
// Load balancing: a CTA owns `spt` * PF_THREADS consecutive output slots whatever the fan-out of the keys behind them
// (skew-proof).  Two threads bisect the scanned match counts for the delta rows of the tile's first and last slot;
// the counts in between are staged in shared memory, where every slot finds its delta row — one global bisection
// per tile instead of one per slot.  Consecutive slots read consecutive trace rows and the same / adjacent delta
// rows, and write consecutive output rows.  The host picks the tile from the match count: one slot per thread
// (spt = 1) spreads a step's few ten thousand matches over every SM; from PF_BIG_TILE_FROM matches on, four slots
// per thread amortise the tile's bisections over more slots (measured faster at q4's match counts on an H100).
constexpr int PF_THREADS = 256, PF_SMEM_ROWS = 3072;
constexpr u64 PF_BIG_TILE_FROM = 1u << 20;
template <class F>
__global__ void
k_probe_fill(Cols D, const i64* wD, u64 nd, BatchRefs tr, int nk, int nvD, int nvT, const u32* lo, const u32* cnt,
             const u32* ki, const u32* exscan, u64 total, int spt, int proj_mode, int delta_is_left, F proj, MCols out,
             i64* out_w) {
  __shared__ u32 s_ex[PF_SMEM_ROWS + 1];
  __shared__ u64 s_rows[2];
  const int tid = threadIdx.x;
  const u64 tile = (u64)spt * PF_THREADS;
  const u64 o0 = (u64)blockIdx.x * tile;
  if (o0 >= total) return;
  const u64 o1 = o0 + tile < total ? o0 + tile : total;
  if (tid < 2) {   // largest i with exscan[i] <= target
    const u64 target = tid == 0 ? o0 : o1 - 1;
    u64 a = 0, b = nd;
    while (b - a > 1) {
      const u64 mid = (a + b) >> 1;
      if (exscan[mid] <= target) a = mid; else b = mid;
    }
    s_rows[tid] = a;
  }
  __syncthreads();
  const u64 row_lo = s_rows[0], row_hi = s_rows[1];
  const u64 nr = row_hi - row_lo + 1;
  const bool staged = nr <= (u64)PF_SMEM_ROWS;
  if (staged)
    for (u64 k = tid; k <= nr; k += PF_THREADS) s_ex[k] = exscan[row_lo + k];
  __syncthreads();
#pragma unroll 1
  for (int qq = 0; qq < spt; qq++) {
    const u64 o = o0 + (u64)qq * PF_THREADS + tid;
    if (o >= o1) break;
    u64 i;
    u32 r;
    if (staged) {
      u32 a = 0, b = (u32)nr;
      while (b - a > 1) {
        const u32 mid = (a + b) >> 1;
        if (s_ex[mid] <= o) a = mid; else b = mid;
      }
      i = row_lo + a;
      r = (u32)(o - s_ex[a]);
    } else {
      u64 a = row_lo, b = row_hi + 1;
      while (b - a > 1) {
        const u64 mid = (a + b) >> 1;
        if (exscan[mid] <= o) a = mid; else b = mid;
      }
      i = a;
      r = (u32)(o - exscan[i]);
    }
    const u64 kbase = (u64)ki[i] * tr.nb;
    // r < the key's total, so the walk stops in a batch with cnt > 0: lo of an empty range (unspecified) is never read
    int bb = 0;
    while (bb < tr.nb - 1 && r >= cnt[kbase + bb]) { r -= cnt[kbase + bb]; bb++; }
    const Cols& T = tr.b[bb].c;
    const u64 t = (u64)lo[kbase + bb] + r;
    u64 row[MAXL];
    i64 wout;
    int nl_out;
    bool ok = true;
    if (proj_mode == 0) {
      nl_out = nk + nvT;
      for (int l = 0; l < nl_out; l++) row[l] = T.c[l][t];
      wout = tr.b[bb].w[t];
    } else {
      u64 key[MAXL], dv[MAXL], tv[MAXL];
      for (int l = 0; l < nk; l++) key[l] = D.c[l][i];
      for (int l = 0; l < nvD; l++) dv[l] = D.c[nk + l][i];
      for (int l = 0; l < nvT; l++) tv[l] = T.c[nk + l][t];
      Env e = delta_is_left ? Env{key, dv, tv} : Env{key, tv, dv};
      ok = project(proj, e, row);
      nl_out = proj.out_schema.n_key_lanes + proj.out_schema.n_val_lanes;
      wout = (i64)((u64)wD[i] * (u64)tr.b[bb].w[t]);
    }
    for (int l = 0; l < nl_out; l++) out.c[l][o] = row[l];
    out_w[o] = ok ? wout : 0;
  }
}

// Sum over one trace batch of the weight of the *exact* row (all L lanes).
__global__ void k_lookup_add(Cols D, u64 nd, Cols T, const i64* wT, u64 nt, int L, Flips f, i64* acc) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nd) return;
  u64 q[MAXL];
  for (int l = 0; l < L; l++) q[l] = D.c[l][i] ^ f.f[l];
  u64 lo = lower_bound_q(T, 0, nt, q, L, f);
  if (lo < nt && cmp_row_q(T, lo, q, L, f) == 0) acc[i] = (i64)((u64)acc[i] + (u64)wT[lo]);
}

// DistinctIncrementalTotal::eval decision (distinct.rs:196-254).
__global__ void k_distinct_decide(const i64* wD, const i64* oldw, u64 n, u32* keep, i64* neww) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  if (i == n) { keep[n] = 0; return; }
  i64 o = oldw[i], nw = (i64)((u64)o + (u64)wD[i]);
  u32 k = 0;
  i64 w = 0;
  if (o <= 0) { if (nw > 0) { k = 1; w = 1; } }
  else if (nw <= 0) { k = 1; w = -1; }
  keep[i] = k;
  neww[i] = w;
}

// The antijoin's weight of a delta row whose key has acc distinct values on the other side: w·(1 − acc), wrapping
// (join.rs:294-320: self − self ⋈ distinct(other)).  A row whose weight is 0 is dropped.
__global__ void k_antijoin_scale(const i64* wD, const i64* acc, u64 n, u32* keep, i64* neww) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  if (i == n) { keep[n] = 0; return; }
  const i64 w = (i64)((u64)wD[i] * ((u64)1 - (u64)acc[i]));
  keep[i] = w != 0;
  neww[i] = w;
}

// IndexedZSet::distinct (algebra/zset/mod.rs:14-38).
__global__ void k_positive(const i64* w, u64 n, u32* keep, i64* neww) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  if (i == n) { keep[n] = 0; return; }
  keep[i] = w[i] > 0 ? 1u : 0u;
  neww[i] = 1;
}

// SemiJoinStream::eval (semijoin.rs:100-142): weight product with the key set.
__global__ void k_semijoin(Cols P, const i64* wP, u64 np, Cols K, const i64* wK, u64 nkeys, int nk, Flips f, u32* keep,
                           i64* neww) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > np) return;
  if (i == np) { keep[np] = 0; return; }
  u64 q[MAXL];
  for (int l = 0; l < nk; l++) q[l] = P.c[l][i] ^ f.f[l];
  u64 lo = lower_bound_q(K, 0, nkeys, q, nk, f);
  i64 w = 0;
  if (lo < nkeys && cmp_row_q(K, lo, q, nk, f) == 0) w = (i64)((u64)wP[i] * (u64)wK[lo]);
  keep[i] = w != 0;
  neww[i] = w;
}

// cursor.seek(val_bound) of the truncating merge (ordered/mod.rs:652-664,
// 729-734) on flat rows: keep the rows whose value lanes are >= the bound.
struct RowBound { u64 v[MAXL]; };   // value lanes, order-flipped
__global__ void k_vals_ge(Cols C, u64 n, int nk, int nv, RowBound b, Flips f, u32* keep) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  if (i == n) { keep[n] = 0; return; }
  bool ge = true;
  for (int l = 0; l < nv; l++) {
    u64 x = C.c[nk + l][i] ^ f.f[nk + l];
    if (x != b.v[l]) { ge = x > b.v[l]; break; }
  }
  keep[i] = ge ? 1u : 0u;
}

// head flag over the first nk lanes (key boundaries of the flat rows).
__global__ void k_key_heads(Cols C, u64 n, int nk, u32* flags) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  if (i == n) { flags[n] = 0; return; }
  bool head = i == 0;
  if (!head)
    for (int l = 0; l < nk; l++)
      if (C.c[l][i] != C.c[l][i - 1]) { head = true; break; }
  flags[i] = head ? 1u : 0u;
}

// The commands of a set / map input (operator/input.rs:128-166): key lanes, the command word ((seq0 + i) << 1 |
// insert), value lanes (0 for a delete), weight 1.  insert == nullptr: every command inserts.
__global__ void k_upsert_cmds(Cols in, int nk, int nv, const uint8_t* insert, u64 n, u64 seq0, MCols out, i64* out_w) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool ins = insert == nullptr || insert[i] != 0;
  for (int l = 0; l < nk; l++) out.c[l][i] = in.c[l][i];
  out.c[nk][i] = ((seq0 + i) << 1) | (ins ? 1u : 0u);
  for (int l = 0; l < nv; l++) out.c[nk + 1 + l][i] = ins ? in.c[nk + l][i] : 0;
  out_w[i] = 1;
}

// Over commands sorted by (key, command word): each key's last command (input.rs:147-160 keeps it), and among those
// the inserts (command bit 1).  last[n] = ins[n] = 0 for the ordered compaction.
__global__ void k_upsert_last(Cols C, u64 n, int nk, u32* last, u32* ins) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  if (i == n) { last[n] = 0; ins[n] = 0; return; }
  bool is_last = i == n - 1;
  if (!is_last)
    for (int l = 0; l < nk; l++)
      if (C.c[l][i] != C.c[l][i + 1]) { is_last = true; break; }
  last[i] = is_last ? 1u : 0u;
  ins[i] = (is_last && (C.c[nk][i] & 1)) ? 1u : 0u;
}

// ordered compaction: out[pos[i]] = row i for keep[i] != 0
__global__ void k_scatter(Cols in, int L, const i64* w, const u32* keep, const u32* pos, u64 n, MCols out, i64* out_w) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !keep[i]) return;
  u32 o = pos[i];
  for (int l = 0; l < L; l++) out.c[l][o] = in.c[l][i];
  if (out_w) out_w[o] = w[i];
}
__global__ void k_scatter_index(const u32* keep, const u32* pos, u64 n, u64* out, u64 nout) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && keep[i]) out[pos[i]] = i;
  if (i == 0) out[nout] = n;
}
__global__ void k_fill_i64(i64* out, u64 n, i64 v) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = v;
}

__global__ void k_neg(const i64* w, u64 n, i64* out) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (i64)((u64)0 - (u64)w[i]);
}

// Aggregator pick over a gathered, consolidated key group batch G (rows of the
// affected keys, weights summed over the spine's batches, zeros dropped):
// Max = last row of each key (max.rs:36-55), Min = first (min.rs:38-57),
// Fold count / sum (fold.rs:76-96), WeightedCount (aggregate/mod.rs:129-156).
__global__ void k_agg_pick(Cols G, const i64* wG, u64 n, int nk, int nv, int kind, const i64* psum, Flips f, u32* keep,
                           MCols out, int out_nv) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  if (i == n) { keep[n] = 0; return; }
  bool first = i == 0, last = i == n - 1;
  if (!first)
    for (int l = 0; l < nk; l++)
      if (G.c[l][i] != G.c[l][i - 1]) { first = true; break; }
  if (!last)
    for (int l = 0; l < nk; l++)
      if (G.c[l][i] != G.c[l][i + 1]) { last = true; break; }
  u32 k = 0;
  u64 v[MAXL];
  if (kind == DBSP_AGG_MAX) {
    k = last;
    for (int l = 0; l < nv; l++) v[l] = G.c[nk + l][i];
  } else if (kind == DBSP_AGG_MIN) {
    k = first;
    for (int l = 0; l < nv; l++) v[l] = G.c[nk + l][i];
  } else if (kind == DBSP_AGG_FOLD_COUNT || kind == DBSP_AGG_FOLD_SUM) {
    k = last;
    if (last) {
      u64 q[MAXL];
      for (int l = 0; l < nk; l++) q[l] = G.c[l][i] ^ f.f[l];
      u64 start = lower_bound_q(G, 0, i + 1, q, nk, f);
      if (kind == DBSP_AGG_FOLD_COUNT) v[0] = i - start + 1;
      else v[0] = (u64)psum[i] - (start ? (u64)psum[start - 1] : 0ull);
    }
  } else if (kind == DBSP_AGG_WCOUNT) {
    k = 1;
    v[0] = (u64)wG[i];
  } else {   // WCOUNT2: rows (K.., which): sum at which == 0, count at which == 1
    k = first;
    if (first) {
      u64 which = G.c[nk][i];
      bool two = !last;   // a second row of the same key follows
      v[0] = which == 0 ? (u64)wG[i] : 0;
      v[1] = which == 1 ? (u64)wG[i] : (two ? (u64)wG[i + 1] : 0);
    }
  }
  keep[i] = k;
  if (k)
    for (int l = 0; l < out_nv; l++) out.c[l][i] = v[l];
}

// A Fold's two programs as kernel parameters: the step as a dbsp_rowfn (validate.h's fold_step_rowfn) so that
// run_rowfn runs both, and the accumulator's first value.
struct FoldArgs {
  dbsp_rowfn step;
  dbsp_rowfn output;
  u64 init[DBSP_MAX_ACC];
  int n_acc;
};
// Fold (fold.rs:60-75) over a gathered, consolidated key group batch G (the affected keys' rows in value order,
// weights summed over the spine's batches, zeros dropped).  Fold is not associative, so a key is walked serially: the
// thread of the key's first row runs `step` on each of the key's rows in order, then `output`, and writes the output
// lanes and the keep flag at that row.  Every other row gets keep = 0.  Every row of G has a non-zero weight, so every
// key in G is non-empty.
__global__ void k_agg_fold(Cols G, const i64* wG, u64 n, int nk, FoldArgs fa, u32* keep, MCols out, int out_nv) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  if (i == n) { keep[n] = 0; return; }
  bool first = i == 0;
  if (!first)
    for (int l = 0; l < nk; l++)
      if (G.c[l][i] != G.c[l][i - 1]) { first = true; break; }
  if (!first) { keep[i] = 0; return; }
  u64 acc[DBSP_MAX_ACC];
  for (int a = 0; a < fa.n_acc; a++) acc[a] = fa.init[a];
  u64 st[DBSP_MAX_STACK];
  for (u64 r = i; r < n; r++) {
    bool same = true;
    for (int l = 0; l < nk && r > i; l++)
      if (G.c[l][r] != G.c[l][i]) { same = false; break; }
    if (!same) break;
    run_rowfn(fa.step, FoldEnv{G, nk, r, acc, wG[r]}, st);
    if (st[fa.n_acc])
      for (int a = 0; a < fa.n_acc; a++) acc[a] = st[a];
  }
  run_rowfn(fa.output, FoldEnv{G, nk, i, acc, 0}, st);
  keep[i] = st[out_nv] != 0;
  for (int l = 0; l < out_nv; l++) out.c[l][i] = st[l];
}

// Max / Min.  Per key, a walk over the union of the spine batches' value lists from the extreme end — the
// CursorList walk of max.rs:36-55 (backwards from the end) / min.rs:38-57 (forwards): per batch a cursor into the
// key's value range; the candidate is the extreme value under the cursors, its weight the sum over the batches that
// hold it (cursor_list.rs:200-210); a zero sum (the value was retracted by another batch — e.g. a merge still in
// progress holds +1 and -1 in two batches) steps those cursors and tries the next value.  Keys that need more than
// AGG_WALK steps are flagged for the general gather path.
constexpr int AGG_WALK = 64;
__global__ void k_agg_extremum(Cols K, u64 nkeys, int nk, int nv, BatchRefs tr, Flips f, int is_max, u32* keep, MCols outv,
               u64* slow_counter) {
  __shared__ BatchBounds s;
  load_bounds(s, tr, nk, f);
  const u64 base = (u64)blockIdx.x * TB + (threadIdx.x & ~31);   // the keys are distinct and sorted: a warp's 32 keys
  const u64 i = base + (threadIdx.x & 31);
  if (i == nkeys) keep[nkeys] = 0;
  if (base >= nkeys) return;   // whole warps only: the range search below takes every lane of a warp
  const bool active = i < nkeys;
  u64 q[MAXL], best[MAXL];
  if (active)
    for (int l = 0; l < nk; l++) q[l] = K.c[l][i] ^ f.f[l];
  warp_key_span(s, q, (int)min(nkeys - base, (u64)32), nk);
  // the key's value range [lo, hi) in every batch; cur = next candidate position
  u32 lo[MAX_REFS], hi[MAX_REFS];
  for (int b = 0; b < tr.nb; b++) {
    u64 l0, h0;
    warp_key_range(s, tr, b, q, active, nk, f, l0, h0);
    lo[b] = (u32)l0;
    hi[b] = (u32)h0;
  }
  if (!active) return;
  bool have = false, exhausted = false;
  i64 wsum = 0;
  for (int it = 0; it < AGG_WALK; it++) {
    have = false;
    for (int b = 0; b < tr.nb; b++) {
      if (lo[b] >= hi[b]) continue;
      const Cols& T = tr.b[b].c;
      const u64 r = is_max ? (u64)hi[b] - 1 : (u64)lo[b];
      int c = 0;   // cmp(candidate, best) over the value lanes
      u64 cand[MAXL];
      for (int l = 0; l < nv; l++) {
        cand[l] = T.c[nk + l][r] ^ f.f[nk + l];
        if (have && c == 0 && cand[l] != best[l]) c = cand[l] < best[l] ? -1 : 1;
      }
      if (!have || (is_max ? c > 0 : c < 0)) {
        for (int l = 0; l < nv; l++) best[l] = cand[l];
        have = true;
      }
    }
    if (!have) break;   // every cursor ran off its range: the key has no value left
    wsum = 0;
    for (int b = 0; b < tr.nb; b++) {
      if (lo[b] >= hi[b]) continue;
      const Cols& T = tr.b[b].c;
      const u64 r = is_max ? (u64)hi[b] - 1 : (u64)lo[b];
      bool eq = true;
      for (int l = 0; l < nv; l++) eq = eq && ((T.c[nk + l][r] ^ f.f[nk + l]) == best[l]);
      if (eq) {
        wsum = (i64)((u64)wsum + (u64)tr.b[b].w[r]);
        if (is_max) hi[b]--; else lo[b]++;   // step past the candidate
      }
    }
    if (wsum != 0) break;
    if (it == AGG_WALK - 1) exhausted = true;
  }
  u32 k = 0;
  if (exhausted) {
    atomicAdd((unsigned long long*)slow_counter, 1ull);
  } else if (have && wsum != 0) {
    k = 1;
    for (int l = 0; l < nv; l++) outv.c[l][i] = best[l] ^ f.f[nk + l];
  }
  keep[i] = k;
}

// weigh (aggregate/mod.rs:297-323): per row f(k,v)*w; AVG mode emits the
// (sum, count) pair weight as two rows (K,0) / (K,1).
template <class F>
__global__ void k_weigh(Cols B, const i64* w, u64 n, int nk, int nv, F fx, int mode, MCols out, i64* out_w) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  u64 lanes[MAXL];
  for (int l = 0; l < nk + nv; l++) lanes[l] = B.c[l][i];
  Env e{lanes, lanes + nk, lanes + nk};
  u64 fv;
  const bool counted = fn_factor(fx, e, &fv);
  if (mode == DBSP_WEIGH_AVG) {
    for (int l = 0; l < nk; l++) { out.c[l][2 * i] = lanes[l]; out.c[l][2 * i + 1] = lanes[l]; }
    out.c[nk][2 * i] = 0;
    out.c[nk][2 * i + 1] = 1;
    out_w[2 * i] = (i64)(fv * (u64)w[i]);
    out_w[2 * i + 1] = counted ? w[i] : 0;
  } else {
    for (int l = 0; l < nk; l++) out.c[l][i] = lanes[l];
    out_w[i] = (i64)(fv * (u64)w[i]);
  }
}

// lower bounds of several key tuples in one batch (window ranges, truncation)
__global__ void k_lower_bounds(Cols T, u64 nt, int nk, Flips f, const u64* queries, int nq, u64* out) {
  int qi = blockIdx.x * blockDim.x + threadIdx.x;
  if (qi >= nq) return;
  u64 q[MAXL];
  for (int l = 0; l < nk; l++) q[l] = queries[qi * MAXL + l] ^ f.f[l];
  out[qi] = lower_bound_q(T, 0, nt, q, nk, f);
}

__device__ __forceinline__ u64 mix64(u64 x) {
  x += 0x9e3779b97f4a7c15ull;
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}
// shard_batch (communication/shard.rs:165-199): flags[p*(n+1) + i] = (hash(key) % P == p).
// One exclusive scan over the concatenated flag arrays is a *stable* P-way
// partition: shard p's rows follow shard p-1's, each shard keeps its order.
__global__ void k_shard_flags(Cols B, u64 n, int nk, u32 P, u32* flags) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  u32 dest = P;   // i == n: terminator slot of every shard
  if (i < n) {
    u64 h = 0;
    for (int l = 0; l < nk; l++) h = mix64(h ^ B.c[l][i]);
    dest = (u32)(h % P);
  }
  for (u32 p = 0; p < P; p++) flags[(u64)p * (n + 1) + i] = (p == dest) ? 1u : 0u;
}
__global__ void k_shard_scatter(Cols in, int L, const i64* w, const u32* flags, const u32* pos, u64 n, u32 P, MCols out,
                                i64* out_w, u64* bounds) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P) bounds[i] = pos[i * (n + 1)];           // first output slot of shard i
  if (i == P) bounds[P] = pos[(u64)P * (n + 1) - 1]; // total (= n)
  if (i >= n) return;
  for (u32 p = 0; p < P; p++) {
    u64 j = (u64)p * (n + 1) + i;
    if (flags[j]) {
      u32 o = pos[j];
      for (int l = 0; l < L; l++) out.c[l][o] = in.c[l][i];
      out_w[o] = w[i];
    }
  }
}

// ---------------- rolling aggregates (time_series/rolling_aggregate.rs) --------------------------------------------
// Rows are (PK lanes, TS, ...); every kernel below compares the first nk + 1 lanes, flipped like the batch.  TS
// arithmetic is range.rs's, in TS's type (u64, or i64 when sgn): `ts_add` / `ts_sub` are the checked forms (false on
// overflow), `sat_*` the saturating ones.  The offsets of an i64 TS are at most INT64_MAX (validate.h).
struct RollArgs {
  u64 from_off, to_off;
  int from_after, to_after, sgn;
};
__device__ __forceinline__ bool ts_add(u64 x, u64 off, int sgn, u64* r) {
  if (!sgn) { *r = x + off; return *r >= x; }
  if ((i64)x > INT64_MAX - (i64)off) return false;
  *r = (u64)((i64)x + (i64)off);
  return true;
}
__device__ __forceinline__ bool ts_sub(u64 x, u64 off, int sgn, u64* r) {
  if (!sgn) { *r = x - off; return x >= off; }
  if ((i64)x < INT64_MIN + (i64)off) return false;
  *r = (u64)((i64)x - (i64)off);
  return true;
}
__device__ __forceinline__ u64 sat_add(u64 x, u64 off, int sgn) {
  u64 r;
  return ts_add(x, off, sgn, &r) ? r : sgn ? (u64)INT64_MAX : ~0ull;
}
__device__ __forceinline__ u64 sat_sub(u64 x, u64 off, int sgn) {
  u64 r;
  return ts_sub(x, off, sgn, &r) ? r : sgn ? (u64)INT64_MIN : 0ull;
}
// RelRange::range_of (range.rs): false when the range lies outside TS
__device__ __forceinline__ bool range_of(const RollArgs& a, u64 ts, u64* lo, u64* hi) {
  if (a.from_after) { if (!ts_add(ts, a.from_off, a.sgn, lo)) return false; }
  else *lo = sat_sub(ts, a.from_off, a.sgn);
  if (a.to_after) *hi = sat_add(ts, a.to_off, a.sgn);
  else if (!ts_sub(ts, a.to_off, a.sgn, hi)) return false;
  return true;
}
// RelRange::affected_range_of (range.rs): the times whose range holds ts
__device__ __forceinline__ bool affected_of(const RollArgs& a, u64 ts, u64* lo, u64* hi) {
  if (a.to_after) *lo = sat_sub(ts, a.to_off, a.sgn);
  else if (!ts_add(ts, a.to_off, a.sgn, lo)) return false;
  if (a.from_after) { if (!ts_sub(ts, a.from_off, a.sgn, hi)) return false; }
  else *hi = sat_add(ts, a.from_off, a.sgn);
  return true;
}
// The TS rows to gather for the times [a, b]: the union of their ranges and [a, b] itself (whose rows decide
// which times get an output), widened to a hull; both ends are monotone, so sorted intervals stay sorted.
__device__ __forceinline__ u64 gather_lo(const RollArgs& r, u64 a) { return r.from_after ? a : sat_sub(a, r.from_off, r.sgn); }
__device__ __forceinline__ u64 gather_hi(const RollArgs& r, u64 b) { return r.to_after ? sat_add(b, r.to_off, r.sgn) : b; }
__device__ __forceinline__ bool same_lanes(const Cols& C, u64 i, u64 j, int nl) {
  for (int l = 0; l < nl; l++)
    if (C.c[l][i] != C.c[l][j]) return false;
  return true;
}

// 1. Per distinct (pk, ts) of delta (rows 2i, 2i+1): [ts, ts] and affected_range_of(ts) as rows (pk, a, b) of weight
// 1; every other slot gets weight 0, which the consolidation drops.
__global__ void k_roll_intervals(Cols D, u64 n, int nk, RollArgs ra, MCols out, i64* out_w) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u64 ts = D.c[nk][i];
  const bool head = i == 0 || !same_lanes(D, i, i - 1, nk + 1);
  u64 lo = ts, hi = ts;
  const bool aff = head && affected_of(ra, ts, &lo, &hi);
  for (int l = 0; l < nk; l++) out.c[l][2 * i] = out.c[l][2 * i + 1] = D.c[l][i];
  out.c[nk][2 * i] = out.c[nk + 1][2 * i] = ts;
  out.c[nk][2 * i + 1] = lo;
  out.c[nk + 1][2 * i + 1] = hi;
  out_w[2 * i] = head ? 1 : 0;
  out_w[2 * i + 1] = aff ? 1 : 0;
}
// The segmented max-scan of the interval ends (flipped), restarting at each partition: an interval list sorted by
// (pk, a) then covers ts iff ts <= the scanned end of the last interval with a <= ts.
struct SegMax {
  u64 v;
  u32 head;
};
struct SegMaxOp {
  __device__ __forceinline__ SegMax operator()(const SegMax& a, const SegMax& b) const {
    return SegMax{b.head ? b.v : max(a.v, b.v), a.head | b.head};
  }
};
__global__ void k_roll_segs(Cols I, u64 n, int nk, u64 tflip, SegMax* s) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  s[i] = SegMax{I.c[nk + 1][i] ^ tflip, (i == 0 || !same_lanes(I, i, i - 1, nk)) ? 1u : 0u};
}
// 2a. Gather groups: an interval starts a new one when its partition changes or its gather window starts after the
// hull of the windows before it.  flags[n] = 0 for the ordered compaction.
__global__ void k_roll_groups(Cols I, const SegMax* bmax, u64 n, int nk, RollArgs ra, u64 tflip, u32* flags) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  if (i == n) { flags[n] = 0; return; }
  bool head = i == 0 || !same_lanes(I, i, i - 1, nk);
  if (!head) head = (gather_lo(ra, I.c[nk][i]) ^ tflip) > (gather_hi(ra, bmax[i - 1].v ^ tflip) ^ tflip);
  flags[i] = head ? 1u : 0u;
}
// group g = intervals [H[g], H[g+1]): its rows (pk.., lo, hi) of the TS rows to gather
__global__ void k_roll_group_rows(Cols I, const SegMax* bmax, const u64* H, u64 m, int nk, RollArgs ra, u64 tflip, MCols W) {
  u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= m) return;
  const u64 h = H[g], e = H[g + 1] - 1;
  for (int l = 0; l < nk; l++) W.c[l][g] = I.c[l][h];
  W.c[nk][g] = gather_lo(ra, I.c[nk][h]);
  W.c[nk + 1][g] = gather_hi(ra, bmax[e].v ^ tflip);
}
// 2b. Per (group g, batch b): the rows of batch b inside group g, by two binary searches; cnt[nb * m] = 0.
__global__ void k_roll_range_bounds(Cols W, u64 m, BatchRefs tr, int nk, Flips f, u32* start, u32* cnt) {
  u64 x = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  const u64 total = m * (u64)tr.nb;
  if (x > total) return;
  if (x == total) { cnt[total] = 0; return; }
  const int b = (int)(x / m);
  const u64 g = x - (u64)b * m;
  u64 q[MAXL];
  for (int l = 0; l < nk + 1; l++) q[l] = W.c[l][g] ^ f.f[l];
  const Cols& T = tr.b[b].c;
  const u64 s = lower_bound_q(T, 0, tr.b[b].n, q, nk + 1, f);
  q[nk] = W.c[nk + 1][g] ^ f.f[nk];
  const u64 e = upper_bound_q(T, s, tr.b[b].n, q, nk + 1, f);
  start[x] = (u32)s;
  cnt[x] = (u32)(e - s);
}
// the first output row of every batch's slices (pos[b * m], b = 0 .. nb; the last is the total), in one read-back
__global__ void k_roll_publish(const u32* pos, u64 m, int nb, Mail mail) {
  u64 v[MAX_REFS + 1];
  for (int b = 0; b <= nb; b++) v[b] = pos[(u64)b * m];
  mail_publish(mail, v, nb + 1);
}
// output row o: the (batch, group) slice holding it (the last slice starting at or before o), then a copy of the row
__global__ void k_roll_range_copy(const u32* start, const u32* pos, u64 ns, BatchRefs tr, u64 m, int L, u64 total,
                                  MCols out, i64* out_w) {
  u64 o = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= total) return;
  u64 lo = 0, hi = ns;   // largest x < ns with pos[x] <= o
  while (hi - lo > 1) {
    const u64 mid = (lo + hi) >> 1;
    if (pos[mid] <= o) lo = mid; else hi = mid;
  }
  const int b = (int)(lo / m);
  const u64 r = start[lo] + (o - pos[lo]);
  for (int l = 0; l < L; l++) out.c[l][o] = tr.b[b].c.c[l][r];
  out_w[o] = tr.b[b].w[r];
}
// whether (pk, ts) of row `row` of R lies in an affected interval of I (sorted by (pk, a), ends max-scanned)
__device__ __forceinline__ bool roll_member(const Cols& I, const SegMax* bmax, u64 nI, const Cols& R, u64 row, int nk,
                                            const Flips& f) {
  u64 q[MAXL];
  for (int l = 0; l < nk + 1; l++) q[l] = R.c[l][row] ^ f.f[l];
  const u64 k = upper_bound_q(I, 0, nI, q, nk + 1, f);
  if (k == 0) return false;
  for (int l = 0; l < nk; l++)
    if (I.c[l][k - 1] != R.c[l][row]) return false;
  return q[nk] <= bmax[k - 1].v;
}
// 4. the old outputs at the affected times, negated (keep[n] = 0 for the ordered compaction)
__global__ void k_roll_retract(Cols O, const i64* wO, u64 n, Cols I, const SegMax* bmax, u64 nI, int nk, Flips f,
                               u32* keep, i64* neww) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  if (i == n) { keep[n] = 0; return; }
  keep[i] = roll_member(I, bmax, nI, O, i, nk, f) ? 1u : 0u;
  neww[i] = (i64)((u64)0 - (u64)wO[i]);
}
// 3a. LINEAR: per gathered row, f(pk, v) * weight per output lane (0 for a row whose keep flag is 0), for the scan.
// V is G's value lanes after TS, so G's columns are shifted for the row function's LVAL.
__global__ void k_roll_terms(Cols V, const i64* w, u64 n, int nk, dbsp_rowfn fn, int n_agg, i64* terms) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  u64 st[DBSP_MAX_STACK];
  run_rowfn(fn, ColEnv{V, nk, i}, st);
  const bool keep = st[n_agg] != 0;
  for (int l = 0; l < n_agg; l++) terms[(u64)l * n + i] = (i64)(keep ? st[l] * (u64)w[i] : 0);
}
// 3b. MAX / MIN: the better of two rows of G by their V lanes (lanes v0 .. v0 + nvv), ties to the first
__device__ __forceinline__ u32 roll_better(const Cols& G, u32 i, u32 j, int v0, int nvv, const Flips& f, int is_max) {
  for (int l = v0; l < v0 + nvv; l++) {
    const u64 a = G.c[l][i] ^ f.f[l], b = G.c[l][j] ^ f.f[l];
    if (a != b) return ((a > b) == (is_max != 0)) ? i : j;
  }
  return i;
}
constexpr int RMQ_BLK = 32;
__device__ __forceinline__ u32 roll_scan(const Cols& G, u32 lo, u32 hi, int v0, int nvv, const Flips& f, int is_max) {
  u32 best = lo;   // rows [lo, hi], lo <= hi
  for (u32 r = lo + 1; r <= hi; r++) best = roll_better(G, best, r, v0, nvv, f, is_max);
  return best;
}
// the sparse table's level 0: the best row of each 32-row block
__global__ void k_roll_rmq_base(Cols G, u64 n, int v0, int nvv, Flips f, int is_max, u32* t0) {
  u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (j * RMQ_BLK >= n) return;
  t0[j] = roll_scan(G, (u32)(j * RMQ_BLK), (u32)min(n - 1, j * RMQ_BLK + RMQ_BLK - 1), v0, nvv, f, is_max);
}
// level k from level k - 1: entry j covers blocks [j, j + 2^k)
__global__ void k_roll_rmq_level(Cols G, const u32* prev, u32* cur, u64 nblk, u64 half, int v0, int nvv, Flips f,
                                 int is_max) {
  u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (j + 2 * half > nblk) return;
  cur[j] = roll_better(G, prev[j], prev[j + half], v0, nvv, f, is_max);
}
struct RollOut {
  int kind, n_agg, nvv;
  const i64* psum;   // LINEAR: n_agg prefix sums of n rows each
  const u32* rmq;    // MAX / MIN: levels of nblk entries each
  u64 nblk;
};
// 3. Per first row of a (pk, ts) group of G that is an affected time with a row of positive weight and a range: the
// window's rows [l, r) in G by two binary searches, then its aggregate; out lanes (ts, some, agg..), keep[n] = 0.
__global__ void k_roll_out(Cols G, const i64* wG, u64 n, Cols I, const SegMax* bmax, u64 nI, int nk, Flips f,
                           RollArgs ra, RollOut ro, u32* keep, MCols out) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  if (i == n) { keep[n] = 0; return; }
  keep[i] = 0;
  if (i > 0 && same_lanes(G, i, i - 1, nk + 1)) return;
  const u64 ts = G.c[nk][i];
  u64 lo, hi;
  if (!range_of(ra, ts, &lo, &hi) || !roll_member(I, bmax, nI, G, i, nk, f)) return;
  bool pos = false;
  for (u64 j = i; j < n && !pos && (j == i || same_lanes(G, j, i, nk + 1)); j++) pos = wG[j] > 0;
  if (!pos) return;
  u64 q[MAXL];
  for (int l = 0; l < nk; l++) q[l] = G.c[l][i] ^ f.f[l];
  q[nk] = lo ^ f.f[nk];
  const u64 l0 = lower_bound_q(G, 0, n, q, nk + 1, f);
  q[nk] = hi ^ f.f[nk];
  const u64 r0 = upper_bound_q(G, l0, n, q, nk + 1, f);
  const bool some = l0 < r0;
  keep[i] = 1;
  out.c[0][i] = ts;
  out.c[1][i] = some ? 1 : 0;
  if (ro.kind == DBSP_ROLLING_LINEAR) {
    for (int l = 0; l < ro.n_agg; l++) {
      const i64* p = ro.psum + (u64)l * n;
      out.c[2 + l][i] = some ? (u64)p[r0 - 1] - (l0 ? (u64)p[l0 - 1] : 0ull) : 0ull;
    }
    return;
  }
  if (!some) {
    for (int l = 0; l < ro.nvv; l++) out.c[2 + l][i] = 0;
    return;
  }
  const int v0 = nk + 1, is_max = ro.kind == DBSP_ROLLING_MAX;
  const u32 a = (u32)l0, b = (u32)(r0 - 1), ba = a / RMQ_BLK, bb = b / RMQ_BLK;
  u32 best;
  if (bb - ba <= 1) {
    best = roll_scan(G, a, b, v0, ro.nvv, f, is_max);
  } else {
    best = roll_scan(G, a, (ba + 1) * RMQ_BLK - 1, v0, ro.nvv, f, is_max);
    best = roll_better(G, best, roll_scan(G, bb * RMQ_BLK, b, v0, ro.nvv, f, is_max), v0, ro.nvv, f, is_max);
    const u32 nb = bb - ba - 1, k = 31 - __clz(nb);   // blocks ba+1 .. bb-1: two overlapping entries of level k
    const u32* t = ro.rmq + (u64)k * ro.nblk;
    best = roll_better(G, best, roll_better(G, t[ba + 1], t[bb - (1u << k)], v0, ro.nvv, f, is_max), v0, ro.nvv, f, is_max);
  }
  for (int l = 0; l < ro.nvv; l++) out.c[2 + l][i] = G.c[v0 + l][best];
}

inline unsigned blocks(u64 n) { return (unsigned)((n + TB - 1) / TB); }
// Row indices, offsets and scans of the operator kernels are 32-bit: reject (never wrap) anything larger.
#define ROWS32(n, what)                                                                        \
  do {                                                                                         \
    if ((u64)(n) >= 0xffffffffull) {                                                           \
      set_error(std::string(what) + ": 2^32-1 or more rows in one batch; split the batch");   \
      return DBSP_ERR_UNSUPPORTED;                                                             \
    }                                                                                          \
  } while (0)
#define CHECK_P(c, msg)                                   \
  do {                                                    \
    if (!(c)) { set_error(msg); return DBSP_ERR_INVALID; } \
  } while (0)

}  // namespace

// ============================ host side =======================================

// Temporary unsorted row store (L lanes + weights) of capacity cap.
struct TmpRows {
  BufP buf;
  MCols c;
  i64* w = nullptr;
  Cols cc() const {
    Cols r;
    for (int l = 0; l < MAXL; l++) r.c[l] = c.c[l];
    return r;
  }
};
static int32_t tmp_alloc(Ctx* ctx, int L, u64 cap, TmpRows* t) {
  u64 c = (cap + 32) & ~31ull;
  if (c == 0) c = 32;
  TRY(dev_alloc(ctx, (size_t)c * 8 * (L + 1), &t->buf));
  u64* base = (u64*)t->buf->p;
  for (int l = 0; l < MAXL; l++) t->c.c[l] = l < L ? base + (size_t)l * c : nullptr;
  t->w = (i64*)(base + (size_t)L * c);
  return DBSP_OK;
}

int32_t compact_ordered(Ctx* ctx, const dbsp_schema& s, const Cols& in, const i64* w, const u32* keep, u64 n, Batch** out) {
  // keep has n+1 entries (keep[n] == 0)
  ROWS32(n, "compact");
  int L = s.n_key_lanes + s.n_val_lanes;
  BufP pbuf;
  TRY(dev_alloc(ctx, (size_t)(n + 1) * 4, &pbuf));
  u32* pos = (u32*)pbuf->p;
  const Mail mail = mail_begin(ctx);
  TRY(exclusive_scan_u32(ctx, keep, pos, n, &mail));
  u64 nout64;
  TRY(mail_finish(ctx, mail, &nout64, 1));
  const u32 nout = (u32)nout64;
  if (nout == 0) { *out = batch_new_empty(ctx, s); return DBSP_OK; }
  Batch* b;
  MCols oc;
  i64* ow;
  TRY(batch_alloc(ctx, s, nout, &b, &oc, &ow));
  k_scatter<<<blocks(n), TB, 0, ctx->stream>>>(in, L, w, keep, pos, n, oc, ow);
  LAUNCH_COUNT(ctx);
  *out = b;
  return DBSP_OK;
}

// Drop the rows whose value is below `val_bound` (n_val_lanes u64).  Keys left
// without values vanish with their rows.  Shares the batch when nothing is cut.
int32_t op_truncate_values(Ctx* ctx, const Batch* b, const u64* val_bound, Batch** out) {
  int nk = b->s.n_key_lanes, nv = b->s.n_val_lanes;
  if (b->n == 0 || nv == 0) { batch_ref((Batch*)b); *out = (Batch*)b; return DBSP_OK; }
  Flips f = b->flips();
  RowBound rb;
  for (int l = 0; l < nv; l++) rb.v[l] = val_bound[l] ^ f.f[nk + l];
  u64 n = b->n;
  ROWS32(n, "truncate_values");
  BufP kb;
  TRY(dev_alloc(ctx, (size_t)(n + 1) * 4 * 2, &kb));
  u32* keep = (u32*)kb->p;
  u32* pos = keep + (n + 1);
  {
    ProfScope ps(ctx, KID_COMPACT, n * (u64)nv * 8);
    k_vals_ge<<<blocks(n + 1), TB, 0, ctx->stream>>>(b->cols(), n, nk, nv, rb, f, keep);
  }
  LAUNCH_COUNT(ctx);
  const Mail mail = mail_begin(ctx);
  TRY(exclusive_scan_u32(ctx, keep, pos, n, &mail));
  u64 nout64;
  TRY(mail_finish(ctx, mail, &nout64, 1));
  const u32 nout = (u32)nout64;
  if (nout == n) { batch_ref((Batch*)b); *out = (Batch*)b; return DBSP_OK; }
  if (nout == 0) { *out = batch_new_empty(ctx, b->s); return DBSP_OK; }
  Batch* o;
  MCols oc;
  i64* ow;
  TRY(batch_alloc(ctx, b->s, nout, &o, &oc, &ow));
  {
    ProfScope ps(ctx, KID_COMPACT, (n + nout) * (u64)(b->nl() + 1) * 8);
    k_scatter<<<blocks(n), TB, 0, ctx->stream>>>(b->cols(), b->nl(), b->w, keep, pos, n, oc, ow);
  }
  LAUNCH_COUNT(ctx);
  *out = o;
  return DBSP_OK;
}

// Zero-copy view of rows [lo, hi) of a batch (shares its storage).
Batch* batch_slice(Ctx* ctx, const Batch* b, u64 lo, u64 hi) {
  Batch* v = new Batch();
  v->s = b->s;
  v->ctx = ctx;
  v->n = hi - lo;
  for (int l = 0; l < b->nl(); l++) v->col[l] = b->col[l] + lo;
  v->w = b->w + lo;
  v->bufs = b->bufs;
  if (v->n == 0) v->nkeys = 0;
  return v;
}

// Concatenation of consolidated batches whose row ranges are already ordered
// and disjoint (the chunks of a fuelled merge): device-to-device copies only.
// Consumes one reference of each part.
int32_t batch_concat(Ctx* ctx, const dbsp_schema& s, std::vector<Batch*>& parts, Batch** out) {
  std::vector<Batch*> live;
  u64 total = 0;
  for (Batch* p : parts) {
    if (p->n) { live.push_back(p); total += p->n; } else batch_unref(p);
  }
  parts.clear();
  if (live.empty()) { *out = batch_new_empty(ctx, s); return DBSP_OK; }
  if (live.size() == 1) { *out = live[0]; return DBSP_OK; }
  Batch* o;
  MCols oc;
  i64* ow;
  int32_t rc = batch_alloc(ctx, s, total, &o, &oc, &ow);
  if (rc) { for (Batch* p : live) batch_unref(p); return rc; }
  int L = s.n_key_lanes + s.n_val_lanes;
  u64 off = 0;
  for (Batch* p : live) {
    for (int l = 0; l < L; l++)
      cudaMemcpyAsync(oc.c[l] + off, p->col[l], p->n * 8, cudaMemcpyDeviceToDevice, ctx->stream);
    cudaMemcpyAsync(ow + off, p->w, p->n * 8, cudaMemcpyDeviceToDevice, ctx->stream);
    off += p->n;
    batch_unref(p);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { batch_unref(o); set_error(cudaGetErrorString(e)); return DBSP_ERR_CUDA; }
  *out = o;
  return DBSP_OK;
}

// input lanes the closure reads (bit l = lane l of the (key lanes, val lanes) row)
unsigned proj_used_mask(const dbsp_proj& p, int nk_in) {
  unsigned mask = 0;
  auto use = [&](const dbsp_src& s) {
    if (s.kind == DBSP_SRC_KEY) mask |= 1u << s.idx;
    else if (s.kind == DBSP_SRC_LVAL || s.kind == DBSP_SRC_RVAL) mask |= 1u << (nk_in + s.idx);
  };
  int nl = p.out_schema.n_key_lanes + p.out_schema.n_val_lanes;
  for (int l = 0; l < nl; l++) { use(p.out[l].a); if (p.out[l].op >= DBSP_OP_ADD) use(p.out[l].b); }
  for (int i = 0; i < p.n_pred; i++) { use(p.pred[i].a); use(p.pred[i].b); }
  return mask;
}
unsigned rowfn_used_mask(const dbsp_rowfn& f, int nk_in) {
  unsigned mask = 0;
  for (int i = 0; i < f.n_insn; i++) {
    const dbsp_insn& in = f.code[i];
    if (in.op != DBSP_FN_PUSH) continue;
    if (in.kind == DBSP_SRC_KEY) mask |= 1u << in.idx;
    else if (in.kind == DBSP_SRC_LVAL || in.kind == DBSP_SRC_RVAL) mask |= 1u << (nk_in + in.idx);
  }
  return mask;
}
static unsigned used_mask(const dbsp_proj& p, int nk_in) { return proj_used_mask(p, nk_in); }
static unsigned used_mask(const dbsp_rowfn& f, int nk_in) { return rowfn_used_mask(f, nk_in); }
template <class F>
static int used_lanes(const F& p, int n_in_lanes, int nk_in = 0) {
  int c = __builtin_popcount(used_mask(p, nk_in) & ((1u << n_in_lanes) - 1));
  return c;
}
// whether the closure can drop a row: predicates, or a keep flag that is not a non-zero constant
static bool filters(const dbsp_proj& p) { return p.n_pred > 0; }
static bool filters(const dbsp_rowfn& f) {
  const dbsp_insn& last = f.code[f.n_insn - 1];   // validated: at least the keep flag is pushed
  return !(last.op == DBSP_FN_PUSH && last.kind == DBSP_SRC_CONST && last.cst != 0);
}

static u64 fan_out(const dbsp_proj&) { return 1; }
static u64 fan_out(const dbsp_rowfn&) { return 1; }
static u64 fan_out(const RowFnFanout& f) { return f.n_out; }

// project rows of (in cols) through proj, then consolidate.  n input rows; a fan-out projects n * n_out virtual rows.
template <class F>
int32_t project_and_consolidate(Ctx* ctx, const Cols& in, int nk_in, int n_in_lanes, const i64* w, u64 n_in,
                                const F& proj, Batch** out) {
  const dbsp_schema& os = proj.out_schema;
  int Lo = os.n_key_lanes + os.n_val_lanes;
  const u64 n = n_in * fan_out(proj);
  if (n == 0) { *out = batch_new_empty(ctx, os); return DBSP_OK; }
  ROWS32(n, "map_index / flat_map_index");
  const unsigned g = (unsigned)((n + PROJ_ROWS - 1) / PROJ_ROWS);
  const bool filtered = filters(proj);
  const u64 m = n;   // upper bound when a filter is present
  u64* status = nullptr;
  u32* ticket = nullptr;
  u32* d_mw = nullptr;
  BufP cb;
  if (filtered) {
    // status[g] u64 | ticket u32, surviving-row count u32
    TRY(dev_alloc(ctx, (size_t)(g + 1) * 8, &cb));
    CUDA_TRY(cudaMemsetAsync(cb->p, 0, (size_t)(g + 1) * 8, ctx->stream));
    status = (u64*)cb->p;
    ticket = (u32*)(status + g);
    d_mw = ticket + 1;   // stays on the device; the census of consolidate_rows returns it
  }
  const u32* d_m = d_mw;
  TmpRows t;
  TRY(tmp_alloc(ctx, Lo, m, &t));
  {
    // the lanes the closure names read once per input row, the output rows written once (bound: every row of the
    // fan-out survives)
    ProfScope ps(ctx, KID_PROJECT, n_in * (u64)(used_lanes(proj, n_in_lanes, nk_in) + (w ? 1 : 0)) * 8 + m * (u64)(Lo + 1) * 8);
    k_project_rows<<<g, TB, 0, ctx->stream>>>(in, nk_in, w, n, proj, filtered ? 0 : 1, g, ticket, status, t.c, t.w, d_mw);
  }
  LAUNCH_COUNT(ctx);
  return consolidate_rows(ctx, os, t.cc(), t.w, m, &t.buf, out, d_m);
}
template int32_t project_and_consolidate(Ctx*, const Cols&, int, int, const i64*, u64, const dbsp_proj&, Batch**);
template int32_t project_and_consolidate(Ctx*, const Cols&, int, int, const i64*, u64, const dbsp_rowfn&, Batch**);
template int32_t project_and_consolidate(Ctx*, const Cols&, int, int, const i64*, u64, const RowFnFanout&, Batch**);

// Probe `delta` against every batch of `trace` and expand the matches.
// proj == nullptr: gather the matching trace rows unchanged.
// key segment starts of the first nk lanes: kstart[nkeys+1] (u64 row indices),
// plus the key index of every row (u32[n]).
static int32_t key_segments(Ctx* ctx, const Batch* b, int nk, BufP* kstart, BufP* ki, const u32** d_nkeys) {
  // No read-back: the key count stays on the device; buffers and grids downstream are sized by the row count, an
  // upper bound of it.  kstart: u64[n+1] (+ aux words behind it), ki: u32[n].
  ROWS32(b->n, "key_segments");
  const u64 n = b->n;
  const u32 ntiles = (u32)((n + SEG_TILE - 1) / SEG_TILE);
  // kstart[n+1] u64 | status[ntiles] u64 | ticket u32, nkeys u32
  TRY(dev_alloc(ctx, (size_t)(n + 1 + ntiles + 1) * 8, kstart));
  TRY(dev_alloc(ctx, (size_t)(n + 1) * 4, ki));
  u64* ks = (u64*)(*kstart)->p;
  u64* status = ks + (n + 1);
  u32* ticket = (u32*)(status + ntiles);
  u32* nkeys = ticket + 1;
  CUDA_TRY(cudaMemsetAsync(status, 0, (size_t)(ntiles + 1) * 8, ctx->stream));
  {
    ProfScope ps(ctx, KID_PROBE_RANGES, n * (u64)nk * 8 + n * 12);
    k_key_segments<<<ntiles, TB, 0, ctx->stream>>>(b->cols(), n, nk, ntiles, ticket, status, ks, (u32*)(*ki)->p, nkeys);
  }
  LAUNCH_COUNT(ctx);
  *d_nkeys = nkeys;
  return DBSP_OK;
}

// Probe `delta` against (up to MAX_REFS) batches of `trace` and expand the matches.
// proj == nullptr: gather the matching trace rows unchanged.
template <class F>
static int32_t probe_chunk(Ctx* ctx, const Batch* delta, int nk, Batch* const* tb, int nb, const F* proj,
                           int delta_is_left, const dbsp_schema& out_schema, const u64* kstart, const u32* ki,
                           const u32* d_nkeys, Batch** out) {
  cudaStream_t st = ctx->stream;
  const u64 nd = delta->n;
  Flips f = delta->flips();
  BatchRefs refs;
  refs.nb = nb;
  const u64 nkeys = nd;   // upper bound of the distinct keys (the exact count is *d_nkeys)
  u64 trace_rows = 0;
  ROWS32(nd, "join/gather delta");
  for (int b = 0; b < nb; b++) ROWS32(tb[b]->n, "join/gather trace batch");
  for (int b = 0; b < nb; b++) {
    refs.b[b].c = tb[b]->cols();
    refs.b[b].w = tb[b]->w;
    refs.b[b].n = tb[b]->n;
    trace_rows += tb[b]->n;
  }
  BufP kb, rb;
  TRY(dev_alloc(ctx, (size_t)nkeys * nb * 4 * 2 + (size_t)nkeys * 4, &kb));
  u32* lo = (u32*)kb->p;
  u32* cnt = lo + (size_t)nkeys * nb;
  u32* ktot = cnt + (size_t)nkeys * nb;
  // ex[nd+1] u32 (padded to u64) | status[ntiles] u64 | ticket u64
  const u32 ntiles = (u32)((nd + SEG_TILE - 1) / SEG_TILE);
  const size_t ex_u64 = (size_t)(nd + 2) / 2 + 1;
  TRY(dev_alloc(ctx, (ex_u64 + ntiles + 1) * 8, &rb));
  u32* ex = (u32*)rb->p;
  u64* status = (u64*)rb->p + ex_u64;
  u32* ticket = (u32*)(status + ntiles);
  CUDA_TRY(cudaMemsetAsync(status, 0, (size_t)(ntiles + 1) * 8, st));
  {
    // delta keys read once, ranges written once; every bisection step touches one
    // trace key row (bounded by the trace's key bytes)
    u64 lg = 1; while ((1ull << lg) < trace_rows / std::max(nb, 1) + 1) lg++;
    u64 touched = std::min<u64>(nkeys * (u64)nb * 2 * lg, trace_rows) * (u64)std::max(nk, 1) * 8;
    ProfScope ps(ctx, KID_PROBE_RANGES, nkeys * ((u64)nk * 8 + (u64)nb * 8 + 4) + touched);
    const unsigned pg = (unsigned)std::min<u64>(blocks(nkeys), (u64)ctx->sm_count * 16);
    k_probe_keys<<<pg, TB, 0, st>>>(delta->cols(), kstart, d_nkeys, refs, nk, f, lo, cnt, ktot);
  }
  const Mail mail = mail_begin(ctx);
  {
    ProfScope ps(ctx, KID_SCAN, nd * 16);
    k_row_counts_scan<<<ntiles, TB, 0, st>>>(ki, ktot, nd, ntiles, ticket, status, ex, mail);
  }
  ctx->kernel_launches += 2;
  u64 total;
  TRY(mail_finish(ctx, mail, &total, 1));
  if (total >= 0xffffffffull) {
    set_error("join/gather: 2^32-1 or more matches in one step (" + std::to_string(total) + "); feed the delta in smaller batches");
    return DBSP_ERR_UNSUPPORTED;
  }
  if (total == 0) { *out = batch_new_empty(ctx, out_schema); return DBSP_OK; }
  int Lo = out_schema.n_key_lanes + out_schema.n_val_lanes;
  F pj;
  if (proj) pj = *proj; else memset(&pj, 0, sizeof(pj));
  TmpRows t;
  TRY(tmp_alloc(ctx, Lo, total, &t));
  {
    // matched trace rows read once, delta rows read once, output rows written once
    ProfScope ps(ctx, KID_PROBE_FILL, (u64)total * (u64)(tb[0]->nl() - nk + 1) * 8 + nd * (u64)(delta->nl() + 1) * 8 +
                                          (u64)total * (u64)(Lo + 1) * 8);
    const int spt = total >= PF_BIG_TILE_FROM ? 4 : 1;
    const u64 tile = (u64)spt * PF_THREADS;
    k_probe_fill<<<(unsigned)((total + tile - 1) / tile), PF_THREADS, 0, st>>>(delta->cols(), delta->w, nd, refs, nk, delta->nl() - nk, tb[0]->nl() - nk, lo,
                                               cnt, ki, ex, total, spt, proj ? 1 : 0, delta_is_left, pj, t.c, t.w);
  }
  LAUNCH_COUNT(ctx);
  // the Batcher of join.rs:845-858: usually sort-free (ordered slots)
  return consolidate_rows(ctx, out_schema, t.cc(), t.w, total, &t.buf, out);
}

static int32_t merge_tree(Ctx* ctx, std::vector<Batch*>& parts, const dbsp_schema& s, Batch** out);

template <class F>
static int32_t probe_spine(Ctx* ctx, const Batch* delta, int nk, const Spine* trace, const F* proj,
                           int delta_is_left, const dbsp_schema& out_schema, Batch** out) {
  const size_t nb = trace->batches.size();
  if (delta->n == 0 || nb == 0) { *out = batch_new_empty(ctx, out_schema); return DBSP_OK; }
  BufP kstart, ki;
  const u32* nkeys = nullptr;   // device count of the distinct delta keys
  TRY(key_segments(ctx, delta, nk, &kstart, &ki, &nkeys));
  std::vector<Batch*> parts;
  for (size_t b0 = 0; b0 < nb; b0 += MAX_REFS) {
    int cnt = (int)std::min<size_t>(MAX_REFS, nb - b0);
    Batch* part = nullptr;
    int32_t rc = probe_chunk(ctx, delta, nk, trace->batches.data() + b0, cnt, proj, delta_is_left, out_schema,
                             (const u64*)kstart->p, (const u32*)ki->p, nkeys, &part);
    if (rc) { for (Batch* p : parts) batch_unref(p); return rc; }
    parts.push_back(part);
  }
  return merge_tree(ctx, parts, out_schema, out);
}

// JoinTrace::eval (operator/join.rs:732-863)
template <class F>
int32_t op_join_delta_trace(Ctx* ctx, const Batch* delta, const Spine* trace, const F* proj, int delta_is_left,
                            Batch** out) {
  if (delta->s.n_key_lanes != trace->s.n_key_lanes) { set_error("join: key lanes differ"); return DBSP_ERR_INVALID; }
  return probe_spine(ctx, delta, delta->s.n_key_lanes, trace, proj, delta_is_left, proj->out_schema, out);
}

// Join::eval (operator/join.rs:436-473)
template <class F>
int32_t op_join_batches(Ctx* ctx, const Batch* l, const Batch* r, const F* proj, Batch** out) {
  Spine sp;
  sp.s = r->s;
  sp.ctx = ctx;
  if (r->n) sp.batches.push_back((Batch*)r);
  return op_join_delta_trace(ctx, l, &sp, proj, 1, out);
}
template int32_t op_join_delta_trace(Ctx*, const Batch*, const Spine*, const dbsp_proj*, int, Batch**);
template int32_t op_join_delta_trace(Ctx*, const Batch*, const Spine*, const dbsp_rowfn*, int, Batch**);
template int32_t op_join_batches(Ctx*, const Batch*, const Batch*, const dbsp_proj*, Batch**);
template int32_t op_join_batches(Ctx*, const Batch*, const Batch*, const dbsp_rowfn*, Batch**);

// distinct keys (first nk lanes) of a batch as an OrdZSet<K> batch with weight 1
static int32_t distinct_keys(Ctx* ctx, const Batch* b, int nk, Batch** out) {
  dbsp_schema ks;
  memset(&ks, 0, sizeof(ks));
  ks.n_key_lanes = nk;
  for (int l = 0; l < nk; l++) ks.lane_types[l] = b->s.lane_types[l];
  if (b->n == 0) { *out = batch_new_empty(ctx, ks); return DBSP_OK; }
  BufP fb;
  TRY(dev_alloc(ctx, (size_t)(b->n + 1) * 4, &fb));
  u32* flags = (u32*)fb->p;
  k_key_heads<<<blocks(b->n + 1), TB, 0, ctx->stream>>>(b->cols(), b->n, nk, flags);
  LAUNCH_COUNT(ctx);
  return compact_ordered(ctx, ks, b->cols(), b->w, flags, b->n, out);
}

// The stages of AggregateIncremental::eval + Upsert::eval that every aggregator shares
// (operator/aggregate/mod.rs:479-547,600-684; operator/upsert.rs:161-208).
// 2b. the keys' value groups: in_tr's rows of `keys` (nk lanes), weights summed over the batches, zeros dropped
static int32_t gather_groups(Ctx* ctx, const Batch* keys, int nk, const Spine* in_tr, Batch** G) {
  return probe_spine(ctx, keys, nk, in_tr, (const dbsp_proj*)nullptr, 1, in_tr->s, G);
}
// 3. rows (key lanes `key`, new value lanes `vals`) with weight +1 where keep[i] != 0, in row order
static int32_t new_values(Ctx* ctx, const dbsp_schema& os, const u64* const* key, const MCols& vals, const u32* keep,
                          u64 n, Batch** N) {
  const int nk = os.n_key_lanes, nov = os.n_val_lanes;
  Cols src;
  for (int l = 0; l < MAXL; l++) src.c[l] = nullptr;
  for (int l = 0; l < nk; l++) src.c[l] = key[l];
  for (int l = 0; l < nov; l++) src.c[nk + l] = vals.c[l];
  BufP ones;
  TRY(dev_alloc(ctx, (size_t)n * 8, &ones));
  k_fill_i64<<<blocks(n), TB, 0, ctx->stream>>>((i64*)ones->p, n, 1);
  LAUNCH_COUNT(ctx);
  return compact_ordered(ctx, os, src, (const i64*)ones->p, keep, n, N);
}
// 4-5. the keys' current values in the output trace, negated, merged with the new ones (consolidate(+new, -old) per
// key == merge of two consolidated batches).  Takes `keys` and `N`.
static int32_t upsert_keys(Ctx* ctx, Batch* keys, Batch* N, const Spine* out_tr, Batch** out) {
  Batch* O = nullptr;
  int32_t rc = probe_spine(ctx, keys, out_tr->s.n_key_lanes, out_tr, (const dbsp_proj*)nullptr, 1, out_tr->s, &O);
  batch_unref(keys);
  if (rc) { batch_unref(N); return rc; }
  Batch* On = nullptr;
  rc = op_neg(ctx, O, &On);
  batch_unref(O);
  if (rc) { batch_unref(N); return rc; }
  rc = merge_batches(ctx, N, On, out);
  batch_unref(N);
  batch_unref(On);
  return rc;
}

// AggregateIncremental::eval + Upsert::eval
// (operator/aggregate/mod.rs:479-547,600-684; operator/upsert.rs:161-208).
int32_t op_aggregate_delta(Ctx* ctx, const Batch* delta, const Spine* in_tr, const Spine* out_tr, int kind, Batch** out) {
  cudaStream_t st = ctx->stream;
  const dbsp_schema& os = out_tr->s;
  int nk = os.n_key_lanes, nov = os.n_val_lanes;
  if (delta->n == 0) { *out = batch_new_empty(ctx, os); return DBSP_OK; }
  // 1. affected keys
  Batch* keys = nullptr;
  TRY(distinct_keys(ctx, delta, nk, &keys));
  int32_t rc;
  Batch* N = nullptr;
  // 2a. Max / Min: candidates straight from the batches' range ends
  if ((kind == DBSP_AGG_MAX || kind == DBSP_AGG_MIN) && in_tr->batches.size() <= (size_t)MAX_REFS && keys->n) {
    BatchRefs refs;
    refs.nb = (int)in_tr->batches.size();
    for (int b = 0; b < refs.nb; b++) {
      refs.b[b].c = in_tr->batches[b]->cols();
      refs.b[b].w = in_tr->batches[b]->w;
      refs.b[b].n = in_tr->batches[b]->n;
    }
    Flips tf;
    for (int l = 0; l < MAXL; l++)
      tf.f[l] = (l < nk + nov && in_tr->s.lane_types[l] == DBSP_I64) ? 0x8000000000000000ull : 0ull;
    BufP kb;
    TRY(dev_alloc(ctx, (size_t)(keys->n + 1) * 4, &kb));
    TmpRows nvr;
    TRY(tmp_alloc(ctx, nov, keys->n, &nvr));
    u64* slow = ctx->d_scratch + 16;
    CUDA_TRY(cudaMemsetAsync(slow, 0, 8, st));
    {
      u64 lg = 1; while ((1ull << lg) < in_tr->batches[0]->n + 1) lg++;
      ProfScope ps(ctx, KID_AGG_PICK, keys->n * ((u64)nk * 8 + (u64)refs.nb * (lg * 8 + (u64)(nov + 1) * 8) + (u64)nov * 8));
      k_agg_extremum<<<blocks(keys->n + 1), TB, 0, st>>>(keys->cols(), keys->n, nk, nov, refs, tf, kind == DBSP_AGG_MAX,
                                                        (u32*)kb->p, nvr.c, slow);
    }
    LAUNCH_COUNT(ctx);
    u64 nslow;
    TRY(read_back(ctx, slow, 1, &nslow));
    if (nslow == 0) {
      rc = new_values(ctx, os, keys->col, nvr.c, (u32*)kb->p, keys->n, &N);
      if (rc) { batch_unref(keys); return rc; }
    }
  }
  // 2b. general path: the keys' value groups, weights summed over batches
  Batch* G = nullptr;
  if (!N) {
    rc = gather_groups(ctx, keys, nk, in_tr, &G);
    if (rc) { batch_unref(keys); return rc; }
  }
  // 3. aggregate per key -> rows (key, new value) with weight +1
  if (N) {
  } else if (G->n) {
    int gnk = nk, gnv = G->nl() - nk;
    if (kind == DBSP_AGG_WCOUNT2) gnv = 0;   // (K.., which) rows: `which` read as lane nk
    BufP kb, ps;
    TRY(dev_alloc(ctx, (size_t)(G->n + 1) * 4, &kb));
    u32* keep = (u32*)kb->p;
    const i64* psum = nullptr;
    if (kind == DBSP_AGG_FOLD_SUM) {
      TRY(dev_alloc(ctx, (size_t)G->n * 8, &ps));
      TRY(inclusive_scan_i64(ctx, (const i64*)G->col[nk], (i64*)ps->p, G->n));
      psum = (const i64*)ps->p;
    }
    TmpRows nv;
    TRY(tmp_alloc(ctx, nov, G->n, &nv));
    k_agg_pick<<<blocks(G->n + 1), TB, 0, st>>>(G->cols(), G->w, G->n, gnk, gnv, kind, psum, G->flips(), keep, nv.c, nov);
    LAUNCH_COUNT(ctx);
    rc = new_values(ctx, os, G->col, nv.c, keep, G->n, &N);
    if (rc) { batch_unref(keys); batch_unref(G); return rc; }
  } else {
    N = batch_new_empty(ctx, os);
  }
  if (G) batch_unref(G);
  return upsert_keys(ctx, keys, N, out_tr, out);
}

// AggregateIncremental::eval + Upsert::eval with a Fold (operator/aggregate/fold.rs:60-75): the stages above, with
// k_agg_fold as the per-key pick.  A key's walk is serial (Fold is not associative, UnimplementedSemigroup).
int32_t op_aggregate_fold(Ctx* ctx, const Batch* delta, const Spine* in_tr, const Spine* out_tr, const dbsp_fold* fold,
                          Batch** out) {
  const dbsp_schema& os = out_tr->s;
  const int nk = os.n_key_lanes, nov = os.n_val_lanes;
  if (delta->n == 0) { *out = batch_new_empty(ctx, os); return DBSP_OK; }
  Batch* keys = nullptr;
  TRY(distinct_keys(ctx, delta, nk, &keys));
  Batch* G = nullptr;
  int32_t rc = gather_groups(ctx, keys, nk, in_tr, &G);
  if (rc) { batch_unref(keys); return rc; }
  Batch* N = nullptr;
  if (G->n) {
    FoldArgs fa;
    memset(&fa, 0, sizeof(fa));
    fa.step = dbsp_validate::fold_step_rowfn(*fold);
    fa.output = fold->output;
    fa.n_acc = fold->n_acc;
    for (int a = 0; a < fold->n_acc; a++) fa.init[a] = fold->init[a];
    BufP kb;
    TmpRows nv;
    rc = dev_alloc(ctx, (size_t)(G->n + 1) * 4, &kb);
    if (rc == DBSP_OK) rc = tmp_alloc(ctx, nov, G->n, &nv);
    if (rc == DBSP_OK) {
      {
        // G's rows (lanes and weight) read once; each affected key's output lanes written once
        ProfScope ps(ctx, KID_AGG_FOLD, G->n * (u64)(G->nl() + 1) * 8 + keys->n * (u64)nov * 8);
        k_agg_fold<<<blocks(G->n + 1), TB, 0, ctx->stream>>>(G->cols(), G->w, G->n, nk, fa, (u32*)kb->p, nv.c, nov);
      }
      LAUNCH_COUNT(ctx);
      rc = new_values(ctx, os, G->col, nv.c, (u32*)kb->p, G->n, &N);
    }
  } else {
    N = batch_new_empty(ctx, os);
  }
  batch_unref(G);
  if (rc) { batch_unref(keys); return rc; }
  return upsert_keys(ctx, keys, N, out_tr, out);
}

// The command batch of dbsp_upsert_commands: k_upsert_cmds over the (staged) columns, then the consolidation, whose
// order (key, command word) is add_upsert's stable sort by key (input.rs:141-145).  Command words are unique, so no
// two rows are summed.
int32_t op_upsert_commands(Ctx* ctx, const dbsp_schema& table, const Cols& in, const uint8_t* insert, u64 n, u64 seq0,
                           Batch** out) {
  const dbsp_schema cs = dbsp_validate::upsert_command_schema(table);
  if (n == 0) { *out = batch_new_empty(ctx, cs); return DBSP_OK; }
  const int nk = table.n_key_lanes, nv = table.n_val_lanes;
  TmpRows t;
  TRY(tmp_alloc(ctx, nk + 1 + nv, n, &t));
  k_upsert_cmds<<<blocks(n), TB, 0, ctx->stream>>>(in, nk, nv, insert, n, seq0, t.c, t.w);
  LAUNCH_COUNT(ctx);
  return consolidate_rows(ctx, cs, t.cc(), t.w, n, &t.buf, out);
}

// Upsert::eval (operator/upsert.rs:161-208) after add_upsert's last-command-per-key step (input.rs:147-160): the
// affected keys and the +1 rows of the inserting ones by ordered compaction (both stay in key order), then the probe
// of the table's trace, negate and merge that aggregates share.
int32_t op_upsert_delta(Ctx* ctx, const Batch* cmds, const Spine* table, Batch** out) {
  const dbsp_schema& ts = table->s;
  const int nk = ts.n_key_lanes, nv = ts.n_val_lanes;
  const u64 n = cmds->n;
  if (n == 0) { *out = batch_new_empty(ctx, ts); return DBSP_OK; }
  ROWS32(n, "upsert_delta");
  BufP fb;
  TRY(dev_alloc(ctx, (size_t)(n + 1) * 4 * 2, &fb));
  u32* last = (u32*)fb->p;
  u32* ins = last + (n + 1);
  {
    // the key lanes and the command lane read once, the two flag arrays written once
    ProfScope ps(ctx, KID_UPSERT, n * (u64)(nk + 1) * 8 + (n + 1) * 8);
    k_upsert_last<<<blocks(n + 1), TB, 0, ctx->stream>>>(cmds->cols(), n, nk, last, ins);
  }
  LAUNCH_COUNT(ctx);
  dbsp_schema ks;
  memset(&ks, 0, sizeof(ks));
  ks.n_key_lanes = nk;
  for (int l = 0; l < nk; l++) ks.lane_types[l] = ts.lane_types[l];
  Batch* keys = nullptr;
  TRY(compact_ordered(ctx, ks, cmds->cols(), cmds->w, last, n, &keys));
  MCols vals;   // read only: new_values gathers them with the key lanes
  for (int l = 0; l < MAXL; l++) vals.c[l] = l < nv ? const_cast<u64*>(cmds->col[nk + 1 + l]) : nullptr;
  Batch* N = nullptr;
  const int32_t rc = new_values(ctx, ts, cmds->col, vals, ins, n, &N);
  if (rc) { batch_unref(keys); return rc; }
  return upsert_keys(ctx, keys, N, table, out);
}

int32_t op_neg(Ctx* ctx, const Batch* a, Batch** out) {
  if (a->n == 0) { *out = batch_new_empty(ctx, a->s); return DBSP_OK; }
  BufP wb;
  TRY(dev_alloc(ctx, (size_t)a->n * 8, &wb));
  k_neg<<<blocks(a->n), TB, 0, ctx->stream>>>(a->w, a->n, (i64*)wb->p);
  LAUNCH_COUNT(ctx);
  Batch* b = new Batch();
  b->s = a->s;
  b->n = a->n;
  b->ctx = ctx;
  for (int l = 0; l < MAXL; l++) b->col[l] = a->col[l];
  b->w = (const i64*)wb->p;
  b->bufs = a->bufs;   // share the lane storage
  b->bufs.push_back(wb);
  *out = b;
  return DBSP_OK;
}

// weigh (operator/aggregate/mod.rs:297-323)
template <class F>
int32_t op_weigh(Ctx* ctx, const Batch* b, const F* f, int mode, Batch** out) {
  int nk = b->s.n_key_lanes, nv = b->s.n_val_lanes;
  dbsp_schema os;
  memset(&os, 0, sizeof(os));
  os.n_key_lanes = nk + (mode == DBSP_WEIGH_AVG ? 1 : 0);
  for (int l = 0; l < nk; l++) os.lane_types[l] = b->s.lane_types[l];
  if (b->n == 0) { *out = batch_new_empty(ctx, os); return DBSP_OK; }
  u64 m = b->n * (mode == DBSP_WEIGH_AVG ? 2 : 1);
  ROWS32(m, "weigh");
  TmpRows t;
  TRY(tmp_alloc(ctx, os.n_key_lanes, m, &t));
  k_weigh<<<blocks(b->n), TB, 0, ctx->stream>>>(b->cols(), b->w, b->n, nk, nv, *f, mode, t.c, t.w);
  LAUNCH_COUNT(ctx);
  return consolidate_rows(ctx, os, t.cc(), t.w, m, &t.buf, out);
}
template int32_t op_weigh(Ctx*, const Batch*, const dbsp_expr*, int, Batch**);
template int32_t op_weigh(Ctx*, const Batch*, const dbsp_rowfn*, int, Batch**);

// DistinctIncrementalTotal::eval (operator/distinct.rs:196-254)
int32_t op_distinct_delta(Ctx* ctx, const Batch* delta, const Spine* integral, Batch** out) {
  u64 n = delta->n;
  if (n == 0) { *out = batch_new_empty(ctx, delta->s); return DBSP_OK; }
  cudaStream_t st = ctx->stream;
  BufP ab, kb;
  TRY(dev_alloc(ctx, (size_t)n * 8 * 2, &ab));
  TRY(dev_alloc(ctx, (size_t)(n + 1) * 4, &kb));
  i64* acc = (i64*)ab->p;
  i64* neww = acc + n;
  CUDA_TRY(cudaMemsetAsync(acc, 0, (size_t)n * 8, st));
  for (Batch* T : integral->batches) {
    k_lookup_add<<<blocks(n), TB, 0, st>>>(delta->cols(), n, T->cols(), T->w, T->n, delta->nl(), delta->flips(), acc);
    LAUNCH_COUNT(ctx);
  }
  k_distinct_decide<<<blocks(n + 1), TB, 0, st>>>(delta->w, acc, n, (u32*)kb->p, neww);
  LAUNCH_COUNT(ctx);
  return compact_ordered(ctx, delta->s, delta->cols(), neww, (u32*)kb->p, n, out);
}

// antijoin (operator/join.rs:294-320) incrementally, with N(k) the count of k's distinct values on the other side:
// out = delta·(1 − N_t) − trace ⋉ ΔN.  The first term is one lookup per delta row and keeps delta's order, so it
// needs no sort; the second gathers only the trace rows of the keys whose count changed.  Neither expands a key's
// values against the other side's.
int32_t op_antijoin_delta(Ctx* ctx, const Batch* delta, const Spine* trace, const Batch* key_delta,
                          const Spine* key_trace, Batch** out) {
  const int nk = delta->s.n_key_lanes, nv = delta->s.n_val_lanes;
  const u64 n = delta->n;
  Batch* first = nullptr;
  if (n == 0) {
    first = batch_new_empty(ctx, delta->s);
  } else {
    cudaStream_t st = ctx->stream;
    BufP ab, kb;
    TRY(dev_alloc(ctx, (size_t)n * 8 * 2, &ab));
    TRY(dev_alloc(ctx, (size_t)(n + 1) * 4, &kb));
    i64* acc = (i64*)ab->p;
    i64* neww = acc + n;
    CUDA_TRY(cudaMemsetAsync(acc, 0, (size_t)n * 8, st));
    for (Batch* T : key_trace->batches) {
      k_lookup_add<<<blocks(n), TB, 0, st>>>(delta->cols(), n, T->cols(), T->w, T->n, nk, delta->flips(), acc);
      LAUNCH_COUNT(ctx);
    }
    {
      ProfScope ps(ctx, KID_ANTIJOIN, n * (8 + 8 + 8 + 4));   // weights and counts read, weights and flags written
      k_antijoin_scale<<<blocks(n + 1), TB, 0, st>>>(delta->w, acc, n, (u32*)kb->p, neww);
    }
    LAUNCH_COUNT(ctx);
    TRY(compact_ordered(ctx, delta->s, delta->cols(), neww, (u32*)kb->p, n, &first));
  }
  // the identity closure (k, v1) over the trace's rows: weight Δcount · w_trace
  dbsp_proj ident;
  memset(&ident, 0, sizeof(ident));
  ident.out_schema = delta->s;
  for (int l = 0; l < nk + nv; l++) {
    ident.out[l].op = DBSP_OP_COPY;
    ident.out[l].a.kind = l < nk ? DBSP_SRC_KEY : DBSP_SRC_LVAL;
    ident.out[l].a.idx = (uint8_t)(l < nk ? l : l - nk);
  }
  Batch* gathered = nullptr;
  int32_t rc = probe_spine(ctx, key_delta, nk, trace, &ident, 0, delta->s, &gathered);
  if (rc != DBSP_OK) { batch_unref(first); return rc; }
  if (gathered->n == 0) { batch_unref(gathered); *out = first; return DBSP_OK; }
  Batch* neg = nullptr;
  rc = op_neg(ctx, gathered, &neg);
  batch_unref(gathered);
  if (rc == DBSP_OK) {
    rc = merge_batches(ctx, first, neg, out);
    batch_unref(neg);
  }
  batch_unref(first);
  return rc;
}

// IndexedZSet::distinct (algebra/zset/mod.rs:14-38)
int32_t op_stream_distinct(Ctx* ctx, const Batch* b, Batch** out) {
  u64 n = b->n;
  if (n == 0) { *out = batch_new_empty(ctx, b->s); return DBSP_OK; }
  BufP ab, kb;
  TRY(dev_alloc(ctx, (size_t)n * 8, &ab));
  TRY(dev_alloc(ctx, (size_t)(n + 1) * 4, &kb));
  k_positive<<<blocks(n + 1), TB, 0, ctx->stream>>>(b->w, n, (u32*)kb->p, (i64*)ab->p);
  LAUNCH_COUNT(ctx);
  return compact_ordered(ctx, b->s, b->cols(), (i64*)ab->p, (u32*)kb->p, n, out);
}

// SemiJoinStream::eval (operator/semijoin.rs:100-142)
int32_t op_semijoin(Ctx* ctx, const Batch* pairs, const Batch* keys, Batch** out) {
  u64 n = pairs->n;
  // Out: ZSet<Key = (Pairs::Key, Pairs::Val)> (semijoin.rs:47): same flat rows, every lane a key lane
  dbsp_schema os = pairs->s;
  os.n_key_lanes = (uint8_t)pairs->nl();
  os.n_val_lanes = 0;
  if (n == 0 || keys->n == 0) { *out = batch_new_empty(ctx, os); return DBSP_OK; }
  BufP ab, kb;
  TRY(dev_alloc(ctx, (size_t)n * 8, &ab));
  TRY(dev_alloc(ctx, (size_t)(n + 1) * 4, &kb));
  k_semijoin<<<blocks(n + 1), TB, 0, ctx->stream>>>(pairs->cols(), pairs->w, n, keys->cols(), keys->w, keys->n,
                                                   pairs->s.n_key_lanes, pairs->flips(), (u32*)kb->p, (i64*)ab->p);
  LAUNCH_COUNT(ctx);
  return compact_ordered(ctx, os, pairs->cols(), (i64*)ab->p, (u32*)kb->p, n, out);
}

// Balanced merge of consolidated batches; consumes one reference of each part.
static int32_t merge_tree(Ctx* ctx, std::vector<Batch*>& parts, const dbsp_schema& s, Batch** out) {
  int32_t rc = DBSP_OK;
  while (parts.size() > 1) {
    std::vector<Batch*> nxt;
    size_t i = 0;
    for (; i + 1 < parts.size(); i += 2) {
      Batch* m = nullptr;
      if (rc == DBSP_OK) rc = merge_batches(ctx, parts[i], parts[i + 1], &m);
      batch_unref(parts[i]);
      batch_unref(parts[i + 1]);
      if (m) nxt.push_back(m);
    }
    if (i < parts.size()) nxt.push_back(parts[i]);
    parts.swap(nxt);
    if (rc != DBSP_OK) { for (Batch* b : parts) batch_unref(b); parts.clear(); return rc; }
  }
  *out = parts.empty() ? batch_new_empty(ctx, s) : parts[0];
  parts.clear();
  return DBSP_OK;
}

// Window::eval (operator/time_series/window.rs:144-222)
int32_t op_window_delta(Ctx* ctx, const Spine* trace, const Batch* delta, int has_prev, const u64* s0, const u64* e0,
                        const u64* s1, const u64* e1, Batch** out) {
  cudaStream_t st = ctx->stream;
  const dbsp_schema& s = delta->s;
  int nk = s.n_key_lanes, L = delta->nl();
  auto lt = [&](const u64* a, const u64* b) {
    for (int l = 0; l < nk; l++) {
      u64 x = a[l], y = b[l];
      if (s.lane_types[l] == DBSP_I64) { x ^= 1ull << 63; y ^= 1ull << 63; }
      if (x != y) return x < y;
    }
    return false;
  };
  struct Range { const Batch* b; u64 lo, hi; int neg; };
  std::vector<Range> ranges;
  // queries: s0, s1, e0, e1 lower bounds in every batch (+ delta)
  u64 hq[4 * MAXL];
  memset(hq, 0, sizeof(hq));
  for (int l = 0; l < nk; l++) { hq[0 * MAXL + l] = s0[l]; hq[1 * MAXL + l] = s1[l]; hq[2 * MAXL + l] = e0[l]; hq[3 * MAXL + l] = e1[l]; }
  BufP qb;
  TRY(dev_alloc(ctx, sizeof(hq) + 4 * 8, &qb));
  u64* dq = (u64*)qb->p;
  u64* dres = dq + 4 * MAXL;
  CUDA_TRY(cudaMemcpyAsync(dq, hq, sizeof(hq), cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaStreamSynchronize(st));   // hq is a stack buffer
  ctx->h2d_bytes += sizeof(hq);
  auto bounds = [&](const Batch* b, u64* r) -> int32_t {
    if (b->n == 0) { r[0] = r[1] = r[2] = r[3] = 0; return DBSP_OK; }
    k_lower_bounds<<<1, 32, 0, st>>>(b->cols(), b->n, nk, b->flips(), dq, 4, dres);
    LAUNCH_COUNT(ctx);
    return read_back(ctx, dres, 4, r);
  };
  u64 r[4];
  if (has_prev) {
    for (Batch* b : trace->batches) {
      TRY(bounds(b, r));
      u64 ps0 = r[0], ps1 = r[1], pe0 = r[2], pe1 = r[3];
      // region 1: [s0, min(s1, e0))
      u64 hi1 = std::min(ps1, pe0);
      if (hi1 > ps0) ranges.push_back({b, ps0, hi1, 1});
      // shrunk on the right: [e1, e0) when e1 < e0
      if (lt(e1, e0) && pe0 > pe1) ranges.push_back({b, pe1, pe0, 1});
      // region 3: [max(e0, s1), e1)
      u64 from = std::max(pe0, ps1);
      if (pe1 > from) ranges.push_back({b, from, pe1, 0});
    }
  }
  TRY(bounds(delta, r));
  if (r[3] > r[1]) ranges.push_back({delta, r[1], r[3], 0});
  // Every range is a slice of a consolidated batch: a zero-copy view (negated
  // for retractions), and Batch::from_tuples over their union is a merge tree.
  std::vector<Batch*> parts;
  int32_t rc = DBSP_OK;
  for (auto& g : ranges) {
    Batch* v = new Batch();
    v->s = s;
    v->ctx = ctx;
    v->n = g.hi - g.lo;
    for (int l = 0; l < L; l++) v->col[l] = g.b->col[l] + g.lo;
    v->w = g.b->w + g.lo;
    v->bufs = g.b->bufs;
    if (g.neg) {
      Batch* nv = nullptr;
      rc = op_neg(ctx, v, &nv);
      batch_unref(v);
      if (rc) break;
      v = nv;
    }
    parts.push_back(v);
  }
  if (rc != DBSP_OK) { for (Batch* b : parts) batch_unref(b); return rc; }
  return merge_tree(ctx, parts, s, out);
}

// A batch reference released at the end of a scope
struct BatchHold {
  Batch* b = nullptr;
  ~BatchHold() { if (b) batch_unref(b); }
};

// The rows of `sp` inside the m groups W (lanes pk.., lo, hi: rows with that pk and lo <= TS <= hi), weights summed
// over the spine's batches, zero sums dropped.  Per chunk of MAX_REFS batches: the slice bounds of every (batch, group)
// by binary search, their scan, one read-back of every batch's first slot, one copy of the slices; each batch's
// slices are a consolidated view in (pk, ts) order, and a merge tree unites the views.
static int32_t roll_gather(Ctx* ctx, const Spine* sp, int nk, const Cols& W, u64 m, Batch** out) {
  const dbsp_schema& s = sp->s;
  const int L = s.n_key_lanes + s.n_val_lanes;
  const size_t nbat = sp->batches.size();
  std::vector<Batch*> parts;
  auto fail = [&](int32_t rc) { for (Batch* p : parts) batch_unref(p); return rc; };
  // slice starts, counts and their scan are u32: a chunk's rows (which bound its gathered rows) and its slice count
  // stay below 2^32-1, else the call is refused
  auto rows32 = [&](u64 v, const char* what) {
    const dbsp_validate::Refusal r = dbsp_validate::valid_rows32(v, what);
    if (r) set_error(r.text);
    return r ? r.status : DBSP_OK;
  };
  for (size_t b0 = 0; m && b0 < nbat; b0 += MAX_REFS) {
    BatchRefs refs;
    refs.nb = (int)std::min<size_t>(MAX_REFS, nbat - b0);
    u64 rows = 0;
    for (int b = 0; b < refs.nb; b++) {
      const Batch* t = sp->batches[b0 + b];
      refs.b[b] = BatchRef{t->cols(), t->w, t->n};
      rows += t->n;
    }
    if (rows == 0) continue;
    const u64 ns = m * (u64)refs.nb;
    int32_t rc = rows32(rows, "rolling_aggregate: the rows of 16 trace batches");
    if (rc == DBSP_OK) rc = rows32(ns, "rolling_aggregate: groups x trace batches");
    if (rc) return fail(rc);
    BufP sb;
    rc = dev_alloc(ctx, (size_t)(ns + 1) * 4 * 3, &sb);
    if (rc) return fail(rc);
    u32* start = (u32*)sb->p;
    u32* cnt = start + (ns + 1);
    u32* pos = cnt + (ns + 1);
    const Flips f = sp->batches[b0]->flips();
    {
      u64 lg = 1; while ((1ull << lg) < rows / refs.nb + 1) lg++;
      ProfScope ps(ctx, KID_ROLLING, m * (u64)(nk + 2) * 8 + ns * (2 * lg * (u64)(nk + 1) * 8 + 8));
      k_roll_range_bounds<<<blocks(ns + 1), TB, 0, ctx->stream>>>(W, m, refs, nk, f, start, cnt);
    }
    LAUNCH_COUNT(ctx);
    if ((rc = exclusive_scan_u32(ctx, cnt, pos, ns))) return fail(rc);
    const Mail mail = mail_begin(ctx);
    k_roll_publish<<<1, 1, 0, ctx->stream>>>(pos, m, refs.nb, mail);
    LAUNCH_COUNT(ctx);
    u64 first[MAX_REFS + 1];
    if ((rc = mail_finish(ctx, mail, first, refs.nb + 1))) return fail(rc);
    const u64 total = first[refs.nb];
    if (total == 0) continue;
    Batch* all;
    MCols oc;
    i64* ow;
    if ((rc = batch_alloc(ctx, s, total, &all, &oc, &ow))) return fail(rc);
    {
      ProfScope ps(ctx, KID_ROLLING, total * (u64)(L + 1) * 8 * 2);
      k_roll_range_copy<<<blocks(total), TB, 0, ctx->stream>>>(start, pos, ns, refs, m, L, total, oc, ow);
    }
    LAUNCH_COUNT(ctx);
    for (int b = 0; b < refs.nb; b++)
      if (first[b + 1] > first[b]) parts.push_back(batch_slice(ctx, all, first[b], first[b + 1]));
    batch_unref(all);
  }
  return merge_tree(ctx, parts, s, out);
}

// PartitionedRollingAggregate::eval (operator/time_series/rolling_aggregate.rs:436-604) without the radix tree:
// 1. the delta's affected intervals (affected_range_of(ts) and [ts, ts] per distinct (pk, ts)), sorted, their ends
//    max-scanned per partition; 2. in_trace's rows of every time those intervals' windows can read (G); 3. per
//    affected (pk, ts) of G with a positive row and a range, its window in G by binary search, aggregated from a
//    prefix sum (LINEAR: wrapping i64 is a group) or a sparse table over 32-row blocks (MAX / MIN); 4. out_trace's
//    rows at the affected times negated and merged with the new rows.  The work is the delta plus the rows the
//    affected windows hold, never a whole partition.
int32_t op_rolling_aggregate(Ctx* ctx, const Batch* delta, const Spine* in_tr, const Spine* out_tr,
                             const dbsp_rel_range& range, int kind, const dbsp_rowfn* fn, Batch** out) {
  cudaStream_t st = ctx->stream;
  const dbsp_schema& os = out_tr->s;
  const int nk = delta->s.n_key_lanes, nv = delta->s.n_val_lanes, n_agg = os.n_val_lanes - 2;
  const u64 n = delta->n;
  if (n == 0) { *out = batch_new_empty(ctx, os); return DBSP_OK; }
  if (2 * n > (u64)INT32_MAX) {   // the intervals (two per delta row) are scanned with an int count
    set_error("rolling_aggregate: n = " + std::to_string(n) + ": 2^30 or more delta rows in one call; split the delta");
    return DBSP_ERR_UNSUPPORTED;
  }
  const Flips f = delta->flips();
  const u64 tflip = f.f[nk];
  const RollArgs ra{range.from_off, range.to_off, range.from_after ? 1 : 0, range.to_after ? 1 : 0,
                    delta->s.lane_types[nk] == DBSP_I64 ? 1 : 0};
  // 1. affected intervals (pk.., a, b), sorted by the consolidation
  dbsp_schema is;
  memset(&is, 0, sizeof(is));
  is.n_key_lanes = (uint8_t)nk;
  is.n_val_lanes = 2;
  for (int l = 0; l < nk + 1; l++) is.lane_types[l] = delta->s.lane_types[l];
  is.lane_types[nk + 1] = is.lane_types[nk];
  BatchHold I;
  {
    TmpRows t;
    TRY(tmp_alloc(ctx, nk + 2, 2 * n, &t));
    {
      ProfScope ps(ctx, KID_ROLLING, n * (u64)(nk + 1) * 8 + 2 * n * (u64)(nk + 3) * 8);
      k_roll_intervals<<<blocks(n), TB, 0, st>>>(delta->cols(), n, nk, ra, t.c, t.w);
    }
    LAUNCH_COUNT(ctx);
    TRY(consolidate_rows(ctx, is, t.cc(), t.w, 2 * n, &t.buf, &I.b));
  }
  const u64 nI = I.b->n;   // >= 1: every delta row has a head
  BufP segb, tmpb;
  TRY(dev_alloc(ctx, (size_t)nI * sizeof(SegMax) * 2, &segb));
  SegMax* segs = (SegMax*)segb->p;
  SegMax* bmax = segs + nI;
  k_roll_segs<<<blocks(nI), TB, 0, st>>>(I.b->cols(), nI, nk, tflip, segs);
  LAUNCH_COUNT(ctx);
  size_t tmp_bytes = 0;
  CUDA_TRY(cub::DeviceScan::InclusiveScan(nullptr, tmp_bytes, segs, bmax, SegMaxOp(), (int)nI, st));
  TRY(dev_alloc(ctx, tmp_bytes, &tmpb));
  CUDA_TRY(cub::DeviceScan::InclusiveScan(tmpb->p, tmp_bytes, segs, bmax, SegMaxOp(), (int)nI, st));
  LAUNCH_COUNT(ctx);
  // 2. gather groups: intervals whose gather windows overlap, merged
  BufP gb, hb;
  TRY(dev_alloc(ctx, (size_t)(nI + 1) * 4 * 2, &gb));
  TRY(dev_alloc(ctx, (size_t)(nI + 1) * 8, &hb));
  u32* gflag = (u32*)gb->p;
  u32* gpos = gflag + (nI + 1);
  u64* H = (u64*)hb->p;
  k_roll_groups<<<blocks(nI + 1), TB, 0, st>>>(I.b->cols(), bmax, nI, nk, ra, tflip, gflag);
  LAUNCH_COUNT(ctx);
  const Mail gmail = mail_begin(ctx);
  TRY(exclusive_scan_u32(ctx, gflag, gpos, nI, &gmail));
  u64 m;
  TRY(mail_finish(ctx, gmail, &m, 1));
  k_scatter_index<<<blocks(nI), TB, 0, st>>>(gflag, gpos, nI, H, m);
  LAUNCH_COUNT(ctx);
  TmpRows W;
  TRY(tmp_alloc(ctx, nk + 2, m, &W));
  k_roll_group_rows<<<blocks(m), TB, 0, st>>>(I.b->cols(), bmax, H, m, nk, ra, tflip, W.c);
  LAUNCH_COUNT(ctx);
  BatchHold G;
  TRY(roll_gather(ctx, in_tr, nk, W.cc(), m, &G.b));
  // 3. the new rows (pk.., ts, some, agg..) with weight +1
  BatchHold N;
  const u64 ng = G.b->n;
  if (ng == 0) {
    N.b = batch_new_empty(ctx, os);
  } else {
    ROWS32(ng, "rolling_aggregate: gathered rows");
    RollOut ro;
    memset(&ro, 0, sizeof(ro));
    ro.kind = kind;
    ro.n_agg = n_agg;
    ro.nvv = nv - 1;
    const Cols g = G.b->cols();
    BufP pb, rb;
    if (kind == DBSP_ROLLING_LINEAR) {
      Cols V = g;   // LVAL i = G's lane nk + 1 + i (V after TS)
      for (int l = 0; l < nv - 1; l++) V.c[nk + l] = g.c[nk + 1 + l];
      TRY(dev_alloc(ctx, (size_t)ng * 8 * 2 * n_agg, &pb));
      i64* terms = (i64*)pb->p;
      i64* psum = terms + (size_t)ng * n_agg;
      {
        ProfScope ps(ctx, KID_ROLLING, ng * (u64)(used_lanes(*fn, nk + nv - 1, nk) + 1) * 8 + ng * (u64)n_agg * 8);
        k_roll_terms<<<blocks(ng), TB, 0, st>>>(V, G.b->w, ng, nk, *fn, n_agg, terms);
      }
      LAUNCH_COUNT(ctx);
      for (int l = 0; l < n_agg; l++) TRY(inclusive_scan_i64(ctx, terms + (size_t)l * ng, psum + (size_t)l * ng, ng));
      ro.psum = psum;
    } else {
      const u64 nblk = (ng + RMQ_BLK - 1) / RMQ_BLK;
      int levels = 1;
      while ((1ull << levels) <= nblk) levels++;
      TRY(dev_alloc(ctx, (size_t)nblk * levels * 4, &rb));
      u32* tab = (u32*)rb->p;
      const int is_max = kind == DBSP_ROLLING_MAX;
      {
        // G's V lanes read once for the blocks; every level reads two entries and their rows' V lanes
        ProfScope ps(ctx, KID_ROLLING, ng * (u64)(nv - 1) * 8 + (u64)levels * nblk * (4 + 2 * (u64)(nv - 1) * 8 + 8));
        k_roll_rmq_base<<<blocks(nblk), TB, 0, st>>>(g, ng, nk + 1, nv - 1, G.b->flips(), is_max, tab);
        LAUNCH_COUNT(ctx);
        for (int k = 1; k < levels; k++) {
          k_roll_rmq_level<<<blocks(nblk), TB, 0, st>>>(g, tab + (u64)(k - 1) * nblk, tab + (u64)k * nblk, nblk,
                                                        1ull << (k - 1), nk + 1, nv - 1, G.b->flips(), is_max);
          LAUNCH_COUNT(ctx);
        }
      }
      ro.rmq = tab;
      ro.nblk = nblk;
    }
    BufP kb;
    TRY(dev_alloc(ctx, (size_t)(ng + 1) * 4, &kb));
    TmpRows nvr;
    TRY(tmp_alloc(ctx, 2 + n_agg, ng, &nvr));
    {
      // G's PK and TS lanes read for the heads and the searches; per output, its window's two ends (LINEAR) or up to
      // 64 rows and two table entries (MAX / MIN), and its lanes written
      const u64 per = kind == DBSP_ROLLING_LINEAR ? 2 * (u64)n_agg * 8 : (2 * RMQ_BLK + 2) * (u64)(nv - 1) * 8;
      ProfScope ps(ctx, KID_ROLLING, ng * ((u64)(nk + 1) * 8 + 8) + ng * (per + (u64)(2 + n_agg) * 8));
      k_roll_out<<<blocks(ng + 1), TB, 0, st>>>(g, G.b->w, ng, I.b->cols(), bmax, nI, nk, f, ra, ro, (u32*)kb->p, nvr.c);
    }
    LAUNCH_COUNT(ctx);
    TRY(new_values(ctx, os, G.b->col, nvr.c, (u32*)kb->p, ng, &N.b));
  }
  // 4. the old outputs at the affected times, negated, merged with the new ones
  BatchHold O, On;
  TRY(roll_gather(ctx, out_tr, nk, W.cc(), m, &O.b));
  if (O.b->n == 0) { *out = N.b; N.b = nullptr; return DBSP_OK; }
  const u64 no = O.b->n;
  ROWS32(no, "rolling_aggregate: old outputs");
  BufP ob;
  TRY(dev_alloc(ctx, (size_t)(no + 1) * 4 + (size_t)no * 8 + 8, &ob));
  i64* neww = (i64*)ob->p;
  u32* keep = (u32*)(neww + no);
  {
    ProfScope ps(ctx, KID_ROLLING, no * ((u64)(nk + 1) * 8 + 8 + 8 + 4));
    k_roll_retract<<<blocks(no + 1), TB, 0, st>>>(O.b->cols(), O.b->w, no, I.b->cols(), bmax, nI, nk, f, keep, neww);
  }
  LAUNCH_COUNT(ctx);
  TRY(compact_ordered(ctx, os, O.b->cols(), neww, keep, no, &On.b));
  return merge_batches(ctx, N.b, On.b, out);
}

// Map/FlatMap/Index::eval + from_tuples (operator/filter_map.rs:563-577,700-724)
template <class F>
int32_t op_map_index(Ctx* ctx, const Batch* b, const F* proj, Batch** out) {
  return project_and_consolidate(ctx, b->cols(), b->s.n_key_lanes, b->nl(), b->w, b->n, *proj, out);
}
template int32_t op_map_index(Ctx*, const Batch*, const dbsp_proj*, Batch**);
template int32_t op_map_index(Ctx*, const Batch*, const dbsp_rowfn*, Batch**);
template int32_t op_map_index(Ctx*, const Batch*, const RowFnFanout*, Batch**);

// shard_batch (operator/communication/shard.rs:165-199)
int32_t op_shard_partition(Ctx* ctx, const Batch* b, u32 P, Batch** outs) {
  for (u32 p = 0; p < P; p++) outs[p] = nullptr;
  if (b->n == 0) {
    for (u32 p = 0; p < P; p++) outs[p] = batch_new_empty(ctx, b->s);
    return DBSP_OK;
  }
  const u64 n = b->n;
  const int L = b->nl();
  CHECK_P(P <= 64, "shard_partition: at most 64 shards");
  ROWS32((n + 1) * (u64)P, "shard_partition");
  BufP fb;
  const u64 m = (u64)P * (n + 1);
  TRY(dev_alloc(ctx, (size_t)(m + 1) * 4 * 2, &fb));
  u32* flags = (u32*)fb->p;
  u32* pos = flags + (m + 1);
  k_shard_flags<<<blocks(n + 1), TB, 0, ctx->stream>>>(b->cols(), n, b->s.n_key_lanes, P, flags);
  LAUNCH_COUNT(ctx);
  CUDA_TRY(cudaMemsetAsync(flags + m, 0, 4, ctx->stream));
  TRY(exclusive_scan_u32(ctx, flags, pos, m));
  Batch* all;   // one buffer holding the P shards back to back; the shards are views
  MCols oc;
  i64* ow;
  TRY(batch_alloc(ctx, b->s, n, &all, &oc, &ow));
  u64* bounds = ctx->d_scratch + 160;
  k_shard_scatter<<<blocks(std::max<u64>(n, P + 1)), TB, 0, ctx->stream>>>(b->cols(), L, b->w, flags, pos, n, P, oc, ow, bounds);
  LAUNCH_COUNT(ctx);
  u64 hb[65];
  int32_t rc = read_back(ctx, bounds, P + 1, hb);
  if (rc) { batch_unref(all); return rc; }
  for (u32 p = 0; p < P; p++) {
    Batch* v = new Batch();
    v->s = b->s;
    v->ctx = ctx;
    v->n = hb[p + 1] - hb[p];
    for (int l = 0; l < L; l++) v->col[l] = all->col[l] + hb[p];
    v->w = all->w + hb[p];
    v->bufs = all->bufs;
    if (v->n == 0) v->nkeys = 0;
    outs[p] = v;
  }
  batch_unref(all);
  return DBSP_OK;
}

// CSR view: row index of every key's first tuple (OrderedLayer offs,
// trace/layers/ordered/mod.rs:32-44), built on demand.
int32_t batch_build_csr(Ctx* ctx, Batch* b) {
  if (b->nkeys != ~0ull) return DBSP_OK;
  if (b->n == 0) { b->nkeys = 0; return DBSP_OK; }
  ROWS32(b->n, "key_count / download_csr");
  int nk = b->s.n_key_lanes;
  BufP fb, pb;
  TRY(dev_alloc(ctx, (size_t)(b->n + 1) * 4 * 2, &fb));
  u32* flags = (u32*)fb->p;
  u32* pos = flags + (b->n + 1);
  k_key_heads<<<blocks(b->n + 1), TB, 0, ctx->stream>>>(b->cols(), b->n, nk, flags);
  LAUNCH_COUNT(ctx);
  const Mail mail = mail_begin(ctx);
  TRY(exclusive_scan_u32(ctx, flags, pos, b->n, &mail));
  u64 nkeys64;
  TRY(mail_finish(ctx, mail, &nkeys64, 1));
  const u32 nkeys = (u32)nkeys64;
  TRY(dev_alloc(ctx, (size_t)(nkeys + 1) * 8, &pb));
  k_scatter_index<<<blocks(b->n), TB, 0, ctx->stream>>>(flags, pos, b->n, (u64*)pb->p, nkeys);
  LAUNCH_COUNT(ctx);
  b->keystart = pb;
  b->nkeys = nkeys;
  return DBSP_OK;
}

// lower bound of one key tuple in a batch (host value)
int32_t batch_lower_bound(Ctx* ctx, const Batch* b, const u64* key, u64* pos) {
  if (b->n == 0) { *pos = 0; return DBSP_OK; }
  u64 hq[MAXL] = {0};
  for (int l = 0; l < b->s.n_key_lanes; l++) hq[l] = key[l];
  u64* dq = ctx->d_scratch + 96;
  CUDA_TRY(cudaMemcpyAsync(dq, hq, sizeof(hq), cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  k_lower_bounds<<<1, 32, 0, ctx->stream>>>(b->cols(), b->n, b->s.n_key_lanes, b->flips(), dq, 1, ctx->d_scratch + 120);
  LAUNCH_COUNT(ctx);
  return read_back(ctx, ctx->d_scratch + 120, 1, pos);
}
