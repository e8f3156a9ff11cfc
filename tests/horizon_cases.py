"""Backend-generic tests of the stateful operators over long step sequences (30-60 steps), against a
non-incremental model: at step t an operator's output must equal f(I_t) - f(I_{t-1}), where I is the integral of
its inputs and f the whole-Z-set definition of the operator.  f is evaluated only on the keys the step's deltas
touch, in numpy (uint64 lanes, weights wrapping mod 2^64 as in tests/exact_model.py).

By then the traces hold layers in every state of the fuelled spine and the deltas have sizes that move the kernels
onto their other paths.  Each regime asserts that it got there, from the model or from the trace's snapshot rather
than from the operator's output:
* growth: mostly shrinking deltas of 1 to ~300 k rows; probes run while merges are in progress, merges complete
  inside apply_fuel and roll_up, and the trace holds more than 16 batches at some step;
* churn: every step retracts live rows sampled from the integral, and the current max / min of some keys, each row
  once; some steps retract the top (or bottom) 70 values of a key at once, and the model shows that the Max / Min
  walk then meets more than 64 leading candidates whose weights sum to 0;
* hot: one key holds 50 k trace rows (a delta row with more than 1024 matches), and a delta of ~500 k rows of which
  ~0.1 % match (a 1024-slot fill tile that spans more than 3072 delta rows);
* window: monotone bounds, late rows below the window, truncation that slices occupied layers;
* exert: `Spine.exert` at efforts 1, 1000 and 2^40 between steps, then at an effort equal to the fuel a merge still
  owes, changes the schedule and nothing else.

The schedule itself is checked against `SpineModel`, a restatement of the spine's layers in numpy: at checkpoints
(and around every exert and truncation) the CUDA library's snapshot of a trace must hold the model's layers, with
the same kind, the same fuel still owed and the same batch lengths, and the same rows up to 200 k of them.

Two ways in.  `run_ops` owns the spines and calls join_delta_trace / aggregate_delta / distinct_delta in the order
of circuit.py's operators, which lets it snapshot the traces at probe time.  `run_circuit` feeds the same deltas
through a RootCircuit (join, Max, Min, FoldCount, FoldSum, aggregate_linear, average, distinct, antijoin, window).

Given a second backend (`ref`, the oracle when the CUDA library is under test), every output is also compared bit for
bit, and at every checkpoint both libraries' snapshots of the same trace must have the same header.  (Their layers
differ by design once rows cancel: see `schedule_checked`.)  On CUDA the profiler names show which paths ran: Max / Min steps
settled by the walk alone and steps that fell back to the gather, join steps whose consolidation sorted and steps
that were sort-free."""
import os
import tempfile

import numpy as np

import exact_model as em
import refusal_cases as rc
from dbsp_b200 import FoldCount, FoldSum, Max, Min, Proj, RootCircuit, Schema, Spine, capi, key, lval, rval
from exact_model import MIN
from parity_util import assert_batches_equal

# DBSP_HORIZON_STEPS=N runs every regime for N steps instead of its default (longer runs; the coverage assertions
# still apply, so very short runs fail them)
STEPS = int(os.environ.get("DBSP_HORIZON_STEPS", "0"))
I_IN_PROGRESS, I_SINGLE, I_COMPLETE = rc.KINDS["IN_PROGRESS"], rc.KINDS["SINGLE"], rc.KINDS["COMPLETE"]
PF_TILE, PF_SMEM_ROWS, AGG_WALK, MAX_REFS = 1024, 3072, 64, 16   # ops.cu: fill tile, staged rows, walk, batches/launch


# ---- schemas: key ids map monotonically onto the key lanes -------------------------------------------------------
class Pair:
    """Left / right input schemas and the join's lanes.  A key id `kid` (int64) is the key: one i64 lane, or the two
    lanes (kid >> 3 as i64, kid & 7 as u64), whose order is kid's order."""

    def __init__(self, name, sl, sr, lanes):
        self.name, self.sl, self.sr, self.lanes = name, sl, sr, lanes
        src = {"k": sl.key, "l": sl.val, "r": sr.val}
        types = "".join(src[p][i] for p, i in lanes)
        self.out = Schema(types[: sl.nk], types[sl.nk:])
        self.proj = Proj(self.out, [{"k": key, "l": lval, "r": rval}[p](i) for p, i in lanes])

    def key_cols(self, kid):
        kid = np.asarray(kid, np.int64)
        if self.sl.nk == 1:
            return [kid.view(np.uint64)]
        return [(kid >> 3).view(np.uint64), (kid & 7).view(np.uint64)]

    def key_tuple(self, kid):
        return tuple(int(c[0]) for c in self.key_cols([kid]))


PAIRS = {
    "i_i": Pair("i_i", Schema("i", "i"), Schema("i", "i"), [("k", 0), ("l", 0), ("r", 0)]),
    "iu_uiu": Pair("iu_uiu", Schema("iu", "uiu"), Schema("iu", "iuu"), [("k", 0), ("k", 1), ("l", 0), ("l", 1), ("r", 0), ("r", 2)]),
}


def weights(rng, n):
    """+-1 and +-2, and about 1 % MIN or +-2^62: sums that cancel only mod 2^64 (MIN + MIN, 4 x 2^62)."""
    w = rng.choice(np.array([-2, -1, 1, 2], np.int64), n)
    odd = rng.random(n) < 0.01
    w[odd] = rng.choice(np.array([MIN, 1 << 62, -(1 << 62)], np.int64), int(odd.sum()))
    return w


U_SHIFT = 1200   # a u64 value lane 0 holds the drawn value + U_SHIFT: never negative, and 0..199 stay free (BEYOND)


def gen_rows(rng, s, pair, kid, vlo=-1000, vhi=1000):
    """Rows of schema `s` with the given key ids; value lane 0 drawn from [vlo, vhi) (shifted by U_SHIFT when it is
    u64), the others from small ranges."""
    n = len(kid)
    v0 = rng.integers(vlo, vhi, n) + (U_SHIFT if s.val[0] == "u" else 0)
    vals = [v0] + [rng.integers(0 if t == "u" else -3, 4, n) for t in s.val[1:]]
    return pair.key_cols(kid) + [np.asarray(v, np.int64).view(np.uint64) for v in vals], weights(rng, n)


# ---- numpy Z-sets: (uint64 columns, int64 weights), consolidated ----------------------------------------------------
def empty(s):
    return [np.zeros(0, np.uint64) for _ in range(s.nl)], np.zeros(0, np.int64)


def negw(w):
    return (np.uint64(0) - np.asarray(w).view(np.uint64)).view(np.int64)


def plus(s, a, b, sign=1):
    return em.consolidate_np(s, [np.concatenate([x, y]) for x, y in zip(a[0], b[0])],
                             np.concatenate([a[1], b[1] if sign > 0 else negw(b[1])]))


def keyv(cols, nk):
    """One comparable value per row holding its key lanes (the lane itself at one key lane, else a void)."""
    if nk == 1:
        return np.asarray(cols[0], np.uint64)
    a = np.ascontiguousarray(np.stack([np.asarray(c, np.uint64) for c in cols[:nk]], axis=1))
    return a.view(np.dtype((np.void, 8 * nk))).ravel()


def restrict(s, z, kv):
    m = np.isin(keyv(z[0], s.nk), kv)
    return [c[m] for c in z[0]], z[1][m]


def key_heads(s, z):
    n = len(z[1])
    h = np.ones(n, bool)
    if n:
        h[1:] = False
        for c in z[0][: s.nk]:
            h[1:] |= c[1:] != c[:-1]
    return np.flatnonzero(h)


def lt_key(s, cols, bound):
    """Rows whose key lanes are below `bound` (typed lexicographic order)."""
    n = len(cols[0]) if cols else 0
    less, eq = np.zeros(n, bool), np.ones(n, bool)
    for t, c, b in zip(s.key, cols, bound):
        f = em.SIGN if t == "i" else np.uint64(0)
        x, y = c ^ f, np.uint64(em.u64(b)) ^ f
        less |= eq & (x < y)
        eq &= x == y
    return less


# ---- f: the whole-Z-set definitions ---------------------------------------------------------------------------------
def f_join(pair, L, R):
    """Every pair of rows on equal keys, weight w1*w2 mod 2^64."""
    nk = pair.sl.nk
    kl, kr = keyv(L[0], nk), keyv(R[0], nk)
    _, inv = np.unique(np.concatenate([kl, kr]), return_inverse=True)
    cl, cr = inv[: len(kl)], inv[len(kl):]
    order = np.argsort(cr, kind="stable")
    crs = cr[order]
    lo, hi = np.searchsorted(crs, cl, "left"), np.searchsorted(crs, cl, "right")
    cnt = hi - lo
    li = np.repeat(np.arange(len(cl)), cnt)
    start = np.cumsum(cnt) - cnt
    ri = order[lo[li] + (np.arange(len(li)) - start[li])] if len(li) else np.zeros(0, np.int64)
    pick = {"k": lambda i: L[0][i][li], "l": lambda i: L[0][nk + i][li], "r": lambda i: R[0][nk + i][ri]}
    w = (L[1].view(np.uint64)[li] * R[1].view(np.uint64)[ri]).view(np.int64)
    return em.consolidate_np(pair.out, [pick[p](i) for p, i in pair.lanes], w)


def f_agg(s, z, kind):
    """Max / Min: the last / first value of each key; FoldCount: the number of values; FoldSum: their lane 0 summed
    mod 2^64; WCOUNT (aggregate_linear of lval(0)): sum of lane 0 * weight, no row when 0.  Weight 1."""
    cols, w = z
    st = key_heads(s, z)
    nk = s.nk
    if kind in (capi.AGG_MAX, capi.AGG_MIN):
        at = np.append(st[1:], len(w)) - 1 if kind == capi.AGG_MAX and len(st) else st
        return [c[at] for c in cols], np.ones(len(at), np.int64)
    keys = [c[st] for c in cols[:nk]]
    if kind == capi.AGG_FOLD_COUNT:
        v = np.diff(np.append(st, len(w))).astype(np.uint64)
    elif kind == capi.AGG_FOLD_SUM:
        v = np.add.reduceat(cols[nk], st) if len(st) else np.zeros(0, np.uint64)
    else:
        v = np.add.reduceat(cols[nk] * w.view(np.uint64), st) if len(st) else np.zeros(0, np.uint64)
        keep = v != 0
        return [k[keep] for k in keys] + [v[keep]], np.ones(int(keep.sum()), np.int64)
    return keys + [v], np.ones(len(st), np.int64)


def trunc_div(a, b):
    """i64::wrapping_div of two u64 bit patterns, as a u64 bit pattern."""
    sa, sb = em.w64(a), em.w64(b)
    q = abs(sa) // abs(sb)
    return em.u64(q if (sa < 0) == (sb < 0) else -q)


def f_average(s, z):
    """average(lval(0)): sum of lane 0 * weight over sum of weights (mod 2^64), truncating; no row at count 0."""
    cols, w = z
    st = key_heads(s, z)
    if not len(st):
        return [np.zeros(0, np.uint64) for _ in range(s.nk + 1)], np.zeros(0, np.int64)
    tot = np.add.reduceat(cols[s.nk] * w.view(np.uint64), st)
    cnt = np.add.reduceat(w.view(np.uint64), st)
    keep = cnt != 0
    avg = np.array([trunc_div(int(a), int(b)) for a, b in zip(tot[keep], cnt[keep])], np.uint64)
    return [c[st][keep] for c in cols[: s.nk]] + [avg], np.ones(len(avg), np.int64)


def f_distinct(z):
    m = z[1] > 0
    return [c[m] for c in z[0]], np.ones(int(m.sum()), np.int64)


def f_antijoin(pair, L, R):
    """L - L |x| distinct(R) with the closure (k, v1): a row of L keeps weight w * (1 - m), m = the number of
    distinct rows of R on its key."""
    nk = pair.sl.nk
    rk = keyv(f_distinct(R)[0], nk)
    kl = keyv(L[0], nk)
    _, inv = np.unique(np.concatenate([kl, rk]), return_inverse=True)
    m = np.bincount(inv[len(kl):], minlength=len(kl) + len(rk) + 1).astype(np.uint64)[inv[: len(kl)]]
    w = (L[1].view(np.uint64) * (np.uint64(1) - m)).view(np.int64)
    return em.consolidate_np(pair.sl, L[0], w)


def f_window(s, z, bounds):
    lo, hi = bounds
    m = ~lt_key(s, z[0], lo) & lt_key(s, z[0], hi)
    return [c[m] for c in z[0]], z[1][m]


def delta_of(s_out, f, cur, prev):
    return plus(s_out, f(cur), f(prev), -1)


# ---- backends ---------------------------------------------------------------------------------------------------------
def upload(be, s, z):
    return be.batch_from_columns(s, z[0], z[1]) if len(z[1]) else be.batch_empty(s)


def check(got, schema, expect, what, other=None):
    em.assert_download_is(schema, got.download(), expect, what)
    if other is not None:
        assert_batches_equal(got, other, f"{what}: vs the oracle")


def profiled(be, fn):
    """fn() with the per-kernel profile of the call on CUDA ({} elsewhere)."""
    if be.name != "cuda":
        return fn(), {}
    be.profile(True)
    out = fn()
    prof = be.profile_read()
    be.profile(False)
    return out, prof


def launches(prof, name):
    return prof.get(name, {}).get("launches", 0)


def gather_launches(nb):
    """probe_ranges launches of one probe_spine over a trace of nb batches: key segments + one per chunk."""
    return 0 if nb == 0 else 1 + (nb + MAX_REFS - 1) // MAX_REFS


class Coverage:
    def __init__(self):
        self.c = {}

    def add(self, what, n=1):
        self.c[what] = self.c.get(what, 0) + n

    def __getitem__(self, what):
        return self.c.get(what, 0)


def snapshot(bes, spines, tmp, name, cov, what):
    """Save the same trace from every backend; the first backend's file is parsed for coverage.  The others must
    have the same header (schema, bounds, effort).  Their layers are not compared: the two libraries spend merge
    fuel differently (the oracle's merger counts the rows it writes, as the reference's does; the CUDA library
    counts input rows), so after rows cancel their merges complete at different inserts (DESIGN §2)."""
    datas = []
    for i, (be, sp) in enumerate(zip(bes, spines)):
        path = os.path.join(tmp, f"{name}.{i}")
        sp.save(path)
        with open(path, "rb") as f:
            datas.append(f.read())
        os.remove(path)
    snap = rc.parse_snapshot(datas[0])[0]
    inv = [(l["kind"], l["remaining"], [b["n"] for b in l["batches"]]) for l in snap["layers"]]
    for d in datas[1:]:
        other = rc.parse_snapshot(d)[0]
        diff = [f for f in ("nk", "nv", "types", "has_bound", "has_vbound", "effort", "bound", "vbound") if snap[f] != other[f]]
        assert not diff, f"{what}: the libraries' snapshots differ in {diff}"
    for l in snap["layers"]:
        if l["kind"] == I_IN_PROGRESS and all(b["n"] for b in l["batches"]):
            cov.add("probe_in_progress")
        if l["kind"] == I_COMPLETE:
            cov.add("complete")
    return snap, inv


# ---- the spine's schedule, restated ------------------------------------------------------------------------------------
INT64_MAX = (1 << 63) - 1
VACANT = rc.KINDS["VACANT"]


def schedule_checked(be):
    """The CUDA library pays a merge's fuel into an account of input rows, as SpineModel does; the oracle's merger
    counts the rows it writes, as the reference's does, so its layers are not checked against the model."""
    return be.name != "oracle"


class SpineModel:
    """The layers of a trace as the CUDA library schedules them (capi.cu, after spine_fueled.rs: introduce_batch,
    apply_fuel, roll_up, insert_at, tidy_layers, exert, truncate_keys_below), with batches held as numpy Z-sets.
    A merge in progress is a fuel account in input rows: it completes when the fuel paid reaches len(a) + len(b).
    `events` counts where merges completed and what tidy_layers did, for the regimes' coverage."""

    def __init__(self, s):
        self.s, self.layers, self.bound = s, [], None
        self.events = Coverage()

    @staticmethod
    def n(b):
        return 0 if b is None else len(b[1])

    def work(self, l, fuel):
        if l["kind"] != I_IN_PROGRESS:
            return fuel
        if fuel < l["rem"]:
            l["rem"] -= fuel
            return 0
        fuel = INT64_MAX if fuel == INT64_MAX else max(fuel - l["rem"], 1)
        l.update(kind=I_COMPLETE, a=plus(self.s, l["a"], l["b"]), b=None, rem=0)
        return fuel

    def complete(self, i, where):
        l = self.layers[i]
        if l["kind"] == I_IN_PROGRESS:
            self.work(l, INT64_MAX)
            self.events.add(where)
        out = l["a"] if l["kind"] in (I_SINGLE, I_COMPLETE) else None
        self.layers[i] = dict(kind=VACANT, a=None, b=None, rem=0)
        return out

    def insert_at(self, batch, i):
        while len(self.layers) <= i:
            self.layers.append(dict(kind=VACANT, a=None, b=None, rem=0))
        l = self.layers[i]
        if l["kind"] == VACANT:
            l.update(kind=I_SINGLE, a=batch)
        else:
            assert l["kind"] == I_SINGLE, "insert into an incomplete merge"
            if l["a"] is not None and batch is not None:
                l.update(kind=I_IN_PROGRESS, b=batch, rem=self.n(l["a"]) + self.n(batch))
            else:
                l.update(kind=I_COMPLETE, a=l["a"] if l["a"] is not None else batch)

    def apply_fuel(self, fuel_each):
        i = 0
        while i < len(self.layers):
            was = self.layers[i]["kind"]
            self.work(self.layers[i], fuel_each)
            if was == I_IN_PROGRESS and self.layers[i]["kind"] == I_COMPLETE:
                self.events.add("apply_fuel")
            if self.layers[i]["kind"] == I_COMPLETE:
                self.insert_at(self.complete(i, "apply_fuel"), i + 1)
            i += 1

    def roll_up(self, index):
        while len(self.layers) <= index:
            self.layers.append(dict(kind=VACANT, a=None, b=None, rem=0))
        if all(l["kind"] == VACANT for l in self.layers[:index]):
            return
        merged = None
        for i in range(index):
            self.insert_at(merged, i)
            merged = self.complete(i, "roll_up")
        self.insert_at(merged, index)
        if self.layers[index]["kind"] in (I_IN_PROGRESS, I_COMPLETE):
            self.insert_at(self.complete(index, "roll_up"), index + 1)

    def level_len(self, l):
        return self.n(l["a"]) + self.n(l["b"]) if l["kind"] != VACANT else 0

    def tidy(self):
        ls = self.layers
        if not ls or ls[-1]["kind"] != I_SINGLE:
            return
        appropriate = max(self.level_len(ls[-1]) - 1, 0).bit_length()
        while appropriate < len(ls) - 1:
            below = ls[-2]
            if below["kind"] == VACANT or (below["kind"] == I_SINGLE and below["a"] is None):
                del ls[-2]
                self.events.add("tidy_erase")
            elif below["kind"] == I_SINGLE:
                length = len(ls)
                smaller = sum((1 << i) if l["kind"] == I_SINGLE else (2 << i) if l["kind"] in (I_IN_PROGRESS, I_COMPLETE) else 0
                              for i, l in enumerate(ls[: length - 2]))
                if smaller <= (1 << length) // 8:
                    batch = below["a"]
                    del ls[length - 2]
                    self.insert_at(batch, length - 2)
                    self.events.add("tidy_move")
                return
            else:
                return

    def introduce(self, batch, index):
        self.apply_fuel(INT64_MAX if index >= 59 else 8 << index)
        self.roll_up(index)
        self.insert_at(batch, index)
        self.tidy()

    def insert(self, z):
        if not len(z[1]):
            return
        if self.bound is not None:   # the bound cuts the batch, perhaps to nothing; it is inserted all the same
            keep = ~lt_key(self.s, z[0], self.bound)
            z = [c[keep] for c in z[0]], z[1][keep]
        self.introduce(z, max(len(z[1]) - 1, 0).bit_length())
        self.events.c["max_in_progress"] = max(self.events["max_in_progress"],
                                               sum(l["kind"] == I_IN_PROGRESS for l in self.layers))

    def exert(self, effort):
        self.tidy()
        doubles = [l for l in self.layers if l["kind"] in (I_IN_PROGRESS, I_COMPLETE)]
        non_empty = sum(self.level_len(l) > 0 for l in self.layers)
        if doubles or non_empty > 1:
            if doubles:
                self.apply_fuel(effort)
            else:
                self.introduce(None, min(max(effort - 1, 0).bit_length(), 62))

    def truncate_keys_below(self, bound):
        if self.bound is not None and not lt_key(self.s, [np.array([em.u64(x)], np.uint64) for x in self.bound], bound)[0]:
            return
        for l in self.layers:
            self.work(l, INT64_MAX)
        self.bound = bound
        for l in self.layers:
            if l["kind"] in (I_SINGLE, I_COMPLETE) and l["a"] is not None:
                keep = ~lt_key(self.s, l["a"][0], bound)
                l["a"] = [c[keep] for c in l["a"][0]], l["a"][1][keep]

    def in_progress_remaining(self):
        return [l["rem"] for l in self.layers if l["kind"] == I_IN_PROGRESS]

    def assert_same(self, snap, what, rows_up_to=200_000):
        """The library's snapshot has this model's layers: kind, remaining fuel, batch lengths, and the rows when
        the trace holds at most `rows_up_to` of them."""
        got = [(l["kind"], l["remaining"], [b["n"] for b in l["batches"]]) for l in snap["layers"]]
        want = [(l["kind"], l["rem"], [self.n(l["a"]), self.n(l["b"])]) for l in self.layers]
        assert got == want, f"{what}: layers {got} != schedule model {want}"
        if sum(sum(n) for _, _, n in want) > rows_up_to:
            return
        for i, (lg, lw) in enumerate(zip(snap["layers"], self.layers)):
            for bg, bw in zip(lg["batches"], (lw["a"], lw["b"])):
                if bw is not None and len(bw[1]):
                    assert all(np.array_equal(np.array(x, np.uint64), y) for x, y in zip(bg["lanes"], bw[0])), f"{what}: layer {i} rows"
                    assert np.array_equal(np.array(bg["w"], np.int64), bw[1]), f"{what}: layer {i} weights"


# ---- the regimes: deltas per step from the model's integrals --------------------------------------------------------
class Regime:
    steps = 30
    checkpoints = ()   # steps whose traces are snapshotted at probe time (besides every `every`-th)
    every = 6

    def __init__(self, pair, seed, scale=1.0):
        """scale: delta sizes relative to the regime's (the circuit runs use smaller ones)."""
        self.pair, self.rng, self.scale = pair, np.random.default_rng(seed), scale
        self.n = STEPS or self.steps

    def exert(self, t):
        return ()

    def rows(self, s, kid, **kw):
        return em.consolidate_np(s, *gen_rows(self.rng, s, self.pair, kid, **kw))


class Growth(Regime):
    """Mostly shrinking deltas (250 k x 0.7^t, jittered): large layers fill first, then many small inserts pay fuel
    into their merges, so merges stay in progress and the spine gets deep."""
    steps = 45

    def deltas(self, t, L, R):
        p, rng = self.pair, self.rng
        n = max(1, int(self.scale * 250_000 * 0.7 ** t * rng.uniform(0.6, 1.4)))
        m = max(1, int(self.scale * 60_000 * 0.75 ** t * rng.uniform(0.5, 1.5)))
        return self.rows(p.sl, rng.integers(-150_000, 150_000, n)), self.rows(p.sr, rng.integers(-150_000, 150_000, m))

    def assert_coverage(self, cov, cuda):
        assert cov["probe_in_progress"] > 0, cov.c
        assert cov["max_batches"] > MAX_REFS, cov.c
        assert cov["apply_fuel"] > 0 and cov["roll_up"] > 0, cov.c   # merges completed by both, per SpineModel
        if cuda:
            assert cov["join_sorted"] > 0 and cov["join_sort_free"] > 0, cov.c


class Churn(Regime):
    """A bounded integral over 3000 keys whose traces fill with rows that cancel across layers."""
    steps = 40
    every = 4

    def __init__(self, pair, seed, scale=1.0):
        super().__init__(pair, seed, scale)
        self.deep = {}   # step -> [(kid, is_max)] keys whose 70 extreme values are retracted at that step

    def churn(self, s, z, n_new, frac, extra=None):
        """Retract a `frac` sample of the live rows of z, and the rows `extra` marks, each exactly once; insert
        n_new new rows."""
        rng = self.rng
        cols, w = z
        take = rng.random(len(w)) < frac
        if extra is not None:
            take |= extra
        out = em.consolidate_np(s, [c[take] for c in cols], negw(w[take]))
        return plus(s, out, self.rows(s, rng.integers(0, 3000, n_new)))

    def deltas(self, t, L, R):
        p, rng = self.pair, self.rng
        s = p.sl
        extra = np.zeros(len(L[1]), bool)
        # the current max and min row of 40 live keys
        st = key_heads(s, L)
        if len(st):
            ends = np.append(st[1:], len(L[1])) - 1
            pick = rng.choice(len(st), min(40, len(st)), replace=False)
            extra[st[pick]] = extra[ends[pick]] = True
        # every 5th step three keys get 100 values beyond their extreme; 3 steps later the 70 most extreme go at once
        deep = self.deep.pop(t, ())
        kz = keyv(L[0], s.nk)
        for kid, is_max in deep:
            at = np.flatnonzero(kz == keyv(p.key_cols([kid]), s.nk)[0])
            extra[at[-70:] if is_max else at[:70]] = True
        dl = self.churn(s, L, int(rng.integers(500, 6000)), 0.08, extra)
        for kid, is_max in deep:
            self.zero_run = max(getattr(self, "zero_run", 0), zero_run(s, L, dl, plus(s, L, dl), kid, p, is_max))
        if t % 5 == 0 and t + 3 < self.n:
            plan = []
            for j, kid in enumerate(rng.choice(3000, 3, replace=False)):
                is_max = (t // 5 + j) % 2 == 0
                kid = int(kid)
                cols = p.key_cols(np.full(100, kid)) + [beyond(s.val[0], is_max)] + [np.zeros(100, np.uint64) for _ in s.val[1:]]
                dl = plus(s, dl, em.consolidate_np(s, cols, rng.choice(np.array([1, 2], np.int64), 100)))
                plan.append((kid, is_max))
            self.deep[t + 3] = plan
        dr = self.churn(p.sr, R, int(rng.integers(500, 4000)), 0.1)
        return dl, dr

    def assert_coverage(self, cov, cuda):
        assert cov["probe_in_progress"] > 0, cov.c
        assert cov["zero_run"] > AGG_WALK, cov.c
        if cuda:
            assert cov["walk_only"] > 0 and cov["walk_fallback"] > 0, cov.c
            assert cov["join_sorted"] > 0 and cov["join_sort_free"] > 0, cov.c


class Hot(Regime):
    """Key HOT collects 5000 right rows per step for 10 steps (50 k rows); later single left rows on it match all of
    them.  At steps 16 and 17 a left delta of 500 k rows, of which 500 match, is inserted and retracted.  The trace
    holds even key ids only; the rows that do not match have odd ids in the same range, so the matching rows of
    the delta lie far apart."""
    steps = 30
    checkpoints = (12, 16, 17)
    HOT = 8

    def deltas(self, t, L, R):
        p, rng = self.pair, self.rng
        dl = self.rows(p.sl, 2 * rng.integers(0, 10_000, 3000))
        dr = self.rows(p.sr, 2 * rng.integers(0, 10_000, 3000))
        h = int(5000 * self.scale)
        if t < 10:
            cols = p.key_cols(np.full(h, self.HOT)) + [np.arange(t * h, (t + 1) * h, dtype=np.uint64)] + \
                [np.zeros(h, np.uint64) for _ in p.sr.val[1:]]
            dr = plus(p.sr, dr, em.consolidate_np(p.sr, cols, np.ones(h, np.int64)))
        if t in (12, 20, 26):
            dl = plus(p.sl, dl, self.rows(p.sl, np.full(2, self.HOT), vlo=5000 + t * 10, vhi=5000 + t * 10 + 10))
        if t == 16:
            self.sparse = plus(p.sl, self.rows(p.sl, 2 * rng.integers(0, 10_000, int(500_000 * self.scale)) + 1),
                               self.rows(p.sl, 2 * rng.integers(0, 10_000, 500)))
            dl = plus(p.sl, dl, self.sparse)
        if t == 17:
            dl = plus(p.sl, dl, self.sparse, -1)
        return dl, dr

    def assert_coverage(self, cov, cuda):
        assert cov["max_matches"] > PF_TILE, cov.c
        assert cov["max_tile_rows"] > PF_SMEM_ROWS, cov.c


class Exert(Churn):
    """Churn with Spine.exert between steps: the schedule moves, the outputs must not."""
    steps = 30
    every = 3
    EFFORTS = ((1,) * 6, (1000,), (1 << 40,))

    def exert(self, t):
        return self.EFFORTS[t % 3]

    def assert_coverage(self, cov, cuda):
        for e in (1, 1000, 1 << 40, "exact"):
            assert cov[f"exert_moved_{e}"] > 0, cov.c


REGIMES = {"growth": Growth, "churn": Churn, "hot": Hot, "exert": Exert}


def beyond(t, is_max):
    """100 values of value lane 0 above (is_max) or below every value gen_rows draws, in the lane type's order."""
    base = (3000 if is_max else -2100) if t == "i" else (3000 + U_SHIFT if is_max else 0)
    return np.arange(base, base + 100, dtype=np.int64).view(np.uint64)


def zero_run(s, L, dl, L1, kid, pair, is_max):
    """From the model: the number of leading candidates, from the key's extreme value down (max) or up (min), whose
    weight sums to 0 when the rows of L and of the delta dl are walked together (two batches, as in the trace at
    probe time, where dl has not been merged with the older rows yet)."""
    k = keyv(pair.key_cols([kid]), s.nk)
    rows = lambda z: {tuple(int(c[i]) for c in z[0]): int(z[1][i]) for i in np.flatnonzero(np.isin(keyv(z[0], s.nk), k))}
    live, cand = rows(L1), sorted(set(rows(L)) | set(rows(dl)), key=lambda r: tuple(em.typed(t, x) for t, x in zip(s.lanes, r)))
    run = 0
    for r in (reversed(cand) if is_max else cand):
        if r in live:
            break
        run += 1
    return run


def fill_tiles(counts):
    """The delta rows one 1024-slot tile of k_probe_fill spans, per tile, for per-delta-row match counts."""
    ex = np.concatenate([[0], np.cumsum(counts)])
    total = int(ex[-1])
    if total == 0:
        return np.zeros(0, np.int64)
    o0 = np.arange(0, total, PF_TILE)
    o1 = np.minimum(o0 + PF_TILE, total)
    nd = len(counts)
    first = np.searchsorted(ex[:nd], o0, "right") - 1   # largest i with ex[i] <= slot
    last = np.searchsorted(ex[:nd], o1 - 1, "right") - 1
    return last - first + 1


def match_counts(pair, D, T, s_d):
    """Matches of every delta row among the trace's rows on its key (the integral's rows: the regime that asks
    for this inserts each trace row once, so no row is split over batches)."""
    nk = s_d.nk
    kd, kt = keyv(D[0], nk), keyv(T[0], nk)
    _, inv = np.unique(np.concatenate([kd, kt]), return_inverse=True)
    per_key = np.bincount(inv[len(kd):], minlength=len(kd) + len(kt) + 1)
    return per_key[inv[: len(kd)]]


# ---- the operator harness --------------------------------------------------------------------------------------------
class Ops:
    """The stateful operators of circuit.py on spines the test owns: join (right trace inserted before the probe,
    the left trace delayed), Max and Min over the left integral (in_trace = the join's left trace once the delta is
    in), and distinct over the right integral before the delta goes in."""

    def __init__(self, be, pair):
        self.be, self.p = be, pair
        self.lt, self.rt = Spine(be, pair.sl), Spine(be, pair.sr)
        self.out = {capi.AGG_MAX: Spine(be, pair.sl), capi.AGG_MIN: Spine(be, pair.sl)}

    def distinct(self, dr):
        return self.be.distinct_delta(dr, self.rt)

    def join_left(self, dl, dr):
        self.rt.insert(dr)
        return profiled(self.be, lambda: self.be.join_delta_trace(dl, self.rt, self.p.proj, True))

    def join_right(self, dr, dl):
        out = profiled(self.be, lambda: self.be.join_delta_trace(dr, self.lt, self.p.proj, False))
        self.lt.insert(dl)
        return out

    def aggregate(self, dl, kind):
        nb_out = self.out[kind].stats()[1]
        o, prof = profiled(self.be, lambda: self.be.aggregate_delta(dl, self.lt, self.out[kind], kind))
        self.out[kind].insert(o)
        return o, prof, nb_out


def count_join_paths(cov, prof):
    if launches(prof, "probe_fill"):
        sorted_ = launches(prof, "radix_sort") or launches(prof, "chunk_sort")
        cov.add("join_sorted" if sorted_ else "join_sort_free")


def run_ops(be, ref, regime, pair_name, seed=0):
    pair = PAIRS[pair_name]
    reg = REGIMES[regime](pair, seed)
    bes = [be] + ([ref] if ref is not None else [])
    hs = [Ops(b, pair) for b in bes]
    sl, sr = pair.sl, pair.sr
    L, R = empty(sl), empty(sr)
    ml, mr = SpineModel(sl), SpineModel(sr)   # the left and right traces' schedule
    cov = Coverage()

    def layers(spines, model, name, what, c=cov):
        snap = snapshot(bes, spines, tmp, name, c, what)
        if schedule_checked(be):
            model.assert_same(snap[0], what)
        return snap
    with tempfile.TemporaryDirectory() as tmp:
        for t in range(reg.n):
            dl, dr = reg.deltas(t, L, R)
            L1, R1 = plus(sl, L, dl), plus(sr, R, dr)
            kv = np.union1d(keyv(dl[0], sl.nk), keyv(dr[0], sr.nk))
            Lk, Rk, L1k, R1k = (restrict(s, z, kv) for s, z in ((sl, L), (sr, R), (sl, L1), (sr, R1)))
            snap_now = t % reg.every == reg.every - 1 or t in reg.checkpoints
            what = f"{regime}/{pair_name} step {t}"
            bd = [(upload(b, sl, dl), upload(b, sr, dr)) for b in bes]
            # distinct over the right integral before this step's delta
            outs = [h.distinct(d[1]) for h, d in zip(hs, bd)]
            check(outs[0], sr, delta_of(sr, f_distinct, R1k, Rk), f"{what} distinct", outs[1] if ref else None)
            # join: delta_L |x| trace(R incl. delta_R) + delta_R |x| trace(L before delta_L)
            o1 = [h.join_left(d[0], d[1]) for h, d in zip(hs, bd)]
            mr.insert(dr)
            if snap_now:
                layers([h.rt for h in hs], mr, "rt", f"{what} right trace")
            o2 = [h.join_right(d[1], d[0]) for h, d in zip(hs, bd)]
            ml.insert(dl)
            count_join_paths(cov, o1[0][1])
            count_join_paths(cov, o2[0][1])
            outs = [b.merge(a[0], c[0]) for b, a, c in zip(bes, o1, o2)]
            check(outs[0], pair.out, plus(pair.out, f_join(pair, L1k, R1k), f_join(pair, Lk, Rk), -1), f"{what} join",
                  outs[1] if ref else None)
            if len(dl[1]):
                c = match_counts(pair, dl, R1, sl)
                cov.c["max_matches"] = max(cov["max_matches"], int(c.max()))
                tiles = fill_tiles(c)
                cov.c["max_tile_rows"] = max(cov["max_tile_rows"], int(tiles.max()) if len(tiles) else 0)
            if snap_now:
                layers([h.lt for h in hs], ml, "lt", f"{what} left trace")
            cov.c["max_batches"] = max(cov["max_batches"], hs[0].lt.stats()[1], hs[0].rt.stats()[1])
            # Max / Min over the left integral
            for kind in (capi.AGG_MAX, capi.AGG_MIN):
                res = [h.aggregate(d[0], kind) for h, d in zip(hs, bd)]
                o, prof, nb_out = res[0]
                check(o, sl, delta_of(sl, lambda z: f_agg(sl, z, kind), L1k, Lk), f"{what} aggregate {kind}",
                      res[1][0] if ref else None)
                if launches(prof, "agg_pick"):
                    cov.add("walk_fallback" if launches(prof, "probe_ranges") > gather_launches(nb_out) else "walk_only")
            efforts = list(reg.exert(t))
            for i in range(len(efforts) + 1):
                if i == len(efforts):   # then the fuel that settles the left trace's first account exactly
                    if not efforts or not ml.in_progress_remaining():
                        break
                    e, name = ml.in_progress_remaining()[0], "exact"
                else:
                    e = name = efforts[i]
                before = layers([h.lt for h in hs], ml, "ex", f"{what} before exert", Coverage())[1]
                for h in hs:
                    for sp in (h.lt, h.rt):
                        sp.exert(e)
                ml.exert(e)
                mr.exert(e)
                after = layers([h.lt for h in hs], ml, "ex", f"{what} after exert({e})", Coverage())[1]
                if after != before:
                    cov.add(f"exert_moved_{name}")
            L, R = L1, R1
        layers([h.lt for h in hs], ml, "lt", f"{regime}/{pair_name} end, left trace")
        layers([h.rt for h in hs], mr, "rt", f"{regime}/{pair_name} end, right trace")
    cov.c["zero_run"] = getattr(reg, "zero_run", 0)
    for m in (ml, mr):
        for k, v in m.events.c.items():
            cov.c[k] = max(cov[k], v) if k == "max_in_progress" else cov[k] + v
    reg.assert_coverage(cov, be.name == "cuda")
    return cov


class Window(Regime):
    """Keys advance 100 ids per step; a tenth of each delta arrives late, below the window.  Delta sizes are
    log-uniform in [1, 8000], so merges are in progress when the bound rises (the truncation completes them first)."""
    steps = 40

    def deltas(self, t, L, R):
        p, rng = self.pair, self.rng
        n = int(np.exp(rng.uniform(0, np.log(8000))))
        kid = rng.integers(100 * t - 50, 100 * t + 400, n)
        late = rng.random(n) < 0.1
        kid[late] = rng.integers(100 * t - 3000, 100 * t - 300, int(late.sum()))
        return self.rows(p.sl, kid), self.rows(p.sr, rng.integers(100 * t - 500, 100 * t + 400, 200))

    def bounds(self, t):
        return 100 * t - 300, 100 * t + 100

    def assert_coverage(self, cov, cuda):
        assert cov[f"sliced_{I_SINGLE}"] > 0 and cov[f"sliced_{I_COMPLETE}"] > 0, cov.c


REGIMES["window"] = Window
Growth.bounds = lambda self, t: (-150_000 + 6000 * t, -100_000 + 7000 * t)
Churn.bounds = lambda self, t: (60 * t, 800 + 70 * t)
Hot.bounds = lambda self, t: (500 * t, 3000 + 600 * t)


def sliced_layers(s, before, after, bound, cov):
    """Count the layers of `after` (SINGLE or COMPLETE) that a key truncation cut: the layer held rows on both sides
    of the bound before, and holds exactly its rows at or above the bound after."""
    for lb, la in zip(before["layers"], after["layers"]):
        if la["kind"] not in (I_SINGLE, I_COMPLETE) or not la["batches"][0]["n"]:
            continue
        below = above = 0
        for b in lb["batches"]:
            if b["n"]:
                m = lt_key(s, [np.array(c, np.uint64) for c in b["lanes"][: s.nk]], bound)
                below, above = below + int(m.sum()), above + int((~m).sum())
        a = la["batches"][0]
        if below and not lt_key(s, [np.array(c, np.uint64) for c in a["lanes"][: s.nk]], bound).any():
            if lb["kind"] == la["kind"]:
                assert a["n"] == above, (a["n"], above)
            cov.add(f"sliced_{la['kind']}")


def run_window(be, ref, pair_name, seed=0):
    """window_delta on a spine the test owns, as circuit.py's window: probe the delayed trace, insert the delta,
    truncate below the new lower bound.  Expected: the rows of I_t in [s_t, e_t) minus those of I_{t-1} in
    [s_{t-1}, e_{t-1})."""
    pair = PAIRS[pair_name]
    s = pair.sl
    reg = Window(pair, seed)
    bes = [be] + ([ref] if ref is not None else [])
    trs = [Spine(b, s) for b in bes]
    model = SpineModel(s)
    I, prev, cov = empty(s), None, Coverage()
    with tempfile.TemporaryDirectory() as tmp:
        for t in range(reg.n):
            d = reg.deltas(t, I, None)[0]
            lo, hi = reg.bounds(t)
            cur = (pair.key_tuple(lo), pair.key_tuple(hi))
            I1 = plus(s, I, d)
            want = plus(s, f_window(s, I1, cur), f_window(s, I, prev) if prev else empty(s), -1)
            outs = [b.window_delta(tr, upload(b, s, d), prev, cur) for b, tr in zip(bes, trs)]
            check(outs[0], s, want, f"window/{pair_name} step {t}", outs[1] if ref else None)
            for b, tr in zip(bes, trs):
                tr.insert(upload(b, s, d))
            model.insert(d)
            before = snapshot(bes, trs, tmp, "w", cov, f"window step {t} before truncation")[0]
            if schedule_checked(be):
                model.assert_same(before, f"window step {t} before truncation")
            for tr in trs:
                tr.truncate_keys_below(cur[0])
            model.truncate_keys_below(cur[0])
            after = snapshot(bes, trs, tmp, "w", cov, f"window step {t} after truncation")[0]
            if schedule_checked(be):
                model.assert_same(after, f"window step {t} after truncation")
            sliced_layers(s, before, after, cur[0], cov)
            I, prev = I1, cur
    reg.assert_coverage(cov, be.name == "cuda")
    return cov


# ---- circuit runs --------------------------------------------------------------------------------------------------
def run_circuit(be, ref, regime, pair_name, seed=1, scale=0.2):
    """The regime's deltas through a RootCircuit: join, Max, Min, FoldCount, FoldSum, aggregate_linear and average of
    lval(0), distinct of the right input, antijoin, window of the left input."""
    pair = PAIRS[pair_name]
    sl, sr = pair.sl, pair.sr
    reg = REGIMES[regime](pair, seed, scale)
    ks = Schema(sl.key, "u")
    ki = Schema(sl.key, "i")
    bes = [be] + ([ref] if ref is not None else [])
    cur = [{} for _ in bes]
    outs = []
    for b, st in zip(bes, cur):
        c = RootCircuit(b)
        a = c.add_source(lambda st=st: st["a"], sl)
        r = c.add_source(lambda st=st: st["b"], sr)
        w = c.add_source(lambda st=st: st["w"])
        o = {"join": a.join(r, pair.proj), "max": a.aggregate(Max), "min": a.aggregate(Min),
             "count": a.aggregate(FoldCount), "sum": a.aggregate(FoldSum), "linear": a.aggregate_linear(lval(0)),
             "average": a.average(lval(0)), "distinct": r.distinct(), "antijoin": a.antijoin(r), "window": a.window(w)}
        outs.append((c, {k: v.output() for k, v in o.items()}))
    L, R, prev = empty(sl), empty(sr), None
    for t in range(reg.n):
        dl, dr = reg.deltas(t, L, R)
        lo, hi = reg.bounds(t)
        wb = (pair.key_tuple(lo), pair.key_tuple(hi))
        for b, st in zip(bes, cur):
            st.update(a=upload(b, sl, dl), b=upload(b, sr, dr), w=wb)
        for c, _ in outs:
            c.step()
        L1, R1 = plus(sl, L, dl), plus(sr, R, dr)
        kl, kr = keyv(dl[0], sl.nk), keyv(dr[0], sr.nk)
        kv = np.union1d(kl, kr)
        Lk, Rk, L1k, R1k = (restrict(s, z, kv) for s, z in ((sl, L), (sr, R), (sl, L1), (sr, R1)))
        Ll, L1l = restrict(sl, L, kl), restrict(sl, L1, kl)
        Rr, R1r = restrict(sr, R, kr), restrict(sr, R1, kr)
        agg = lambda kind: (lambda z: f_agg(sl, z, kind))
        want = {
            "join": (pair.out, lambda: plus(pair.out, f_join(pair, L1k, R1k), f_join(pair, Lk, Rk), -1)),
            "max": (sl, lambda: delta_of(sl, agg(capi.AGG_MAX), L1l, Ll)),
            "min": (sl, lambda: delta_of(sl, agg(capi.AGG_MIN), L1l, Ll)),
            "count": (ks, lambda: delta_of(ks, agg(capi.AGG_FOLD_COUNT), L1l, Ll)),
            "sum": (ks, lambda: delta_of(ks, agg(capi.AGG_FOLD_SUM), L1l, Ll)),
            "linear": (ki, lambda: delta_of(ki, agg(capi.AGG_WCOUNT), L1l, Ll)),
            "average": (ki, lambda: delta_of(ki, lambda z: f_average(sl, z), L1l, Ll)),
            "distinct": (sr, lambda: delta_of(sr, f_distinct, R1r, Rr)),
            "antijoin": (sl, lambda: plus(sl, f_antijoin(pair, L1k, R1k), f_antijoin(pair, Lk, Rk), -1)),
            "window": (sl, lambda: plus(sl, f_window(sl, L1, wb), f_window(sl, L, prev) if prev else empty(sl), -1)),
        }
        for name, (schema, f) in want.items():
            got = outs[0][1][name].value
            check(got, schema, f(), f"circuit {regime}/{pair_name} step {t} {name}",
                  outs[1][1][name].value if ref else None)
        L, R, prev = L1, R1, wb


def run_snapshot_header(be, ref=None):
    """A trace never bounded saves zeros in its key and value bound fields, so that two saves of the same trace, by
    either library, are equal byte for byte (both fields once held uninitialised memory)."""
    s = Schema("i", "iu")
    bes = [be] + ([ref] if ref is not None else [])
    trs = [Spine(b, s) for b in bes]
    for b, tr in zip(bes, trs):
        tr.insert(b.batch_from_rows(s, [(1, 2, 3, 1), (-5, 0, 7, MIN)]))
    with tempfile.TemporaryDirectory() as tmp:
        snap = snapshot(bes, trs, tmp, "h", Coverage(), "snapshot header")[0]
        datas = []
        for i, tr in enumerate(trs):
            tr.save(os.path.join(tmp, f"b{i}"))
            with open(os.path.join(tmp, f"b{i}"), "rb") as f:
                datas.append(f.read())
    assert all(d == datas[0] for d in datas), "one batch, no merge: the libraries' files must be equal byte for byte"
    assert (snap["has_bound"], snap["has_vbound"]) == (0, 0), snap
    assert snap["bound"] == [0] * 8 and snap["vbound"] == [0] * 8, (snap["bound"], snap["vbound"])


ALL_CASES = {"snapshot_header": run_snapshot_header}
for _p in PAIRS:
    for _r in ("growth", "churn", "hot", "exert"):
        ALL_CASES[f"ops_{_r}_{_p}"] = lambda be, ref=None, r=_r, p=_p: run_ops(be, ref, r, p)
    ALL_CASES[f"ops_window_{_p}"] = lambda be, ref=None, p=_p: run_window(be, ref, p)
    for _r in ("growth", "churn", "hot", "window"):
        ALL_CASES[f"circuit_{_r}_{_p}"] = lambda be, ref=None, r=_r, p=_p: run_circuit(be, ref, r, p)
