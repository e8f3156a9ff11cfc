"""Backend-generic tests of row *shapes* and of the memory a batch sits in: every lane count L = 1..8 with key
splits nk in {0, 1, L//2, L-1, L}, rows without key lanes, and batches that are zero-copy views of other batches.

The kernels specialised by lane count (k_props<L>, k_merge_partition / k_merge_tiles / k_merge_split<L>) run at
sizes around each merge configuration's tile (TILE below: rows per k_merge_tiles block).  The merge kernel stages a
tile with TMA bulk copies only when every lane of an input (and, at <= 2 lanes, its weight array) shares one 16-byte
phase; otherwise it stages row by row with cp.async.  Views reach both: a slice that cuts an odd number of leading
rows puts every lane at the other phase, and the negation of such a slice has its own weight array (so at <= 2 lanes
the weights and the lanes differ in phase).  Run with DBSP_MERGE_NO_TMA=1 (see __main__), every merge stages with
cp.async.

Every case compares the backend's output with tests/exact_model.py; given a second backend (`ref`, the oracle when
the CUDA library is under test) it also compares the two bit for bit."""
import os
import sys
import zlib

import numpy as np

if __name__ == "__main__":   # run as a child process: the repository root and tests/ on the path
    _here = os.path.dirname(os.path.abspath(__file__))
    sys.path[:0] = [os.path.dirname(_here), _here]

import edge_cases as ec
import exact_model as em
import exchange_model as xm
from dbsp_b200 import Proj, Schema, Spine, capi, key, lval, rval
from exact_model import MIN, Z
from parity_util import assert_batches_equal

check = ec.check
TMIN = {"u": 0, "i": MIN}
MODES = ("narrow", "mixed", "full")


def tile(L):
    """Rows per k_merge_tiles block: 1 lane 256 x 9, 2 lanes 128 x 9, 3-6 lanes 256 x 5, 7-8 lanes 256 x 3."""
    return 2304 if L == 1 else 1152 if L == 2 else 1280 if L <= 6 else 768


def sizes(L):
    T = tile(L)
    return [0, 1, T - 1, T, T + 1, 3 * T + 2, BIG]


def shapes():
    """For every L, the key splits {0, 1, L//2, L-1, L}; lane types cycle so that every lane position is `i` in
    some shape."""
    out, j = [], 0
    for L in range(1, 9):
        for nk in sorted({0, 1, L // 2, L - 1, L}):
            t = "".join("i" if (l + j) % 3 == 0 else "u" for l in range(L))
            out.append(Schema(t[:nk], t[nk:]))
            j += 1
    return out


SHAPES = shapes()
BIG = 100_003   # the large size runs in one generation mode per shape (cycling over the shapes), on fewer views


def modes_at(s, n):
    return MODES if n < BIG else (MODES[SHAPES.index(s) % 3] if s in SHAPES else "full",)


def sid(s):
    return f"k{s.key}_v{s.val}"


def seed_of(*parts):
    return zlib.crc32(repr(parts).encode())


# ---- rows ----------------------------------------------------------------------------
def lane_values(rng, s, l, n, mode):
    """Lane l of n generated rows (uint64 bit patterns).  narrow: 5 values (runs, duplicates), except the last lane,
    which spans 4n values so that n distinct rows exist; full: edge_cases.full_lane; mixed: lane 0 full, others
    narrow.  So a width reaches the one-word, two-word and word-by-word packing plans.  Lane 0 never holds one of
    the three smallest values of its type: those are kept for the rows that slices cut (cut_rows)."""
    t = s.lanes[l]
    if mode == "full" or (mode == "mixed" and l == 0):
        x = ec.full_lane(rng, t, n)
    else:
        hi = 4 * n + 8 if l == s.nl - 1 else 5
        x = rng.integers(0, hi, n).astype(np.int64)
        x = (x - hi // 2 if t == "i" else x + 3).view(np.uint64)
    if l == 0:
        floor = np.uint64(em.u64(TMIN[t] + 3))
        flip = em.SIGN if t == "i" else np.uint64(0)
        x = np.where((x ^ flip) < (floor ^ flip), floor, x)
    return x


def small_weights(rng, n):
    """Mostly +-1..3, a tenth from edge_cases' wrapping pool."""
    w = rng.choice(np.array([-3, -2, -1, 1, 2, 3], np.int64), n)
    pick = rng.random(n) < 0.1
    w[pick] = ec.edge_weights(rng, int(pick.sum()))
    w[w == 0] = 1
    return w


def rows(rng, s, n, mode):
    """Exactly n consolidated rows: (sorted uint64 columns, non-zero int64 weights)."""
    m = n + n // 2 + 16
    cols, w = em.consolidate_np(s, [lane_values(rng, s, l, m, mode) for l in range(s.nl)], small_weights(rng, m))
    assert len(w) >= n, (s, n, mode, len(w))
    keep = np.sort(rng.choice(len(w), n, replace=False))
    return [c[keep] for c in cols], w[keep]


def negw(w):
    return (np.uint64(0) - np.asarray(w).view(np.uint64)).view(np.int64)


def concat(s, *parts):
    return [np.concatenate([p[0][l] for p in parts]) for l in range(s.nl)], np.concatenate([p[1] for p in parts])


def ge_lex(cols, types, bound):
    """Rows whose lanes (typed, lexicographic) are >= the bound tuple."""
    n = len(cols[0]) if cols else 0
    res = np.ones(n, bool)
    for c, t, b in zip(cols[::-1], types[::-1], bound[::-1]):
        f = em.SIGN if t == "i" else np.uint64(0)
        x, y = c ^ f, np.uint64(em.u64(b)) ^ f
        res = (x > y) | ((x == y) & res)
    return res


def select(data, m):
    cols, w = data
    return [c[m] for c in cols], w[m]


def z_of(s, data):
    cols, w = data
    return Z(s, zip(*[c.tolist() for c in cols], w.tolist())) if len(w) else Z(s)


# ---- views ---------------------------------------------------------------------------
VIEWS = ("fresh", "cut1", "cut2", "cut3", "neg1", "neg2", "neg3", "reidx")


def cut_rows(s, c):
    """c rows that sort before every generated row (lane 0 = the type's minimum + 0..c-1), weight 1."""
    cols = [np.array([em.u64(TMIN[s.lanes[0]] + j) for j in range(c)], np.uint64)]
    cols += [np.zeros(c, np.uint64) for _ in range(s.nl - 1)]
    return cols, np.ones(c, np.int64)


def view(be, s, data, kind):
    """A batch of schema s holding exactly the consolidated rows `data`, built as `kind`:
      fresh  its own allocation;
      cutC   truncate_keys_below of a batch with C more leading rows: a zero-copy view starting C rows in
             (at nk = 0 the cut is made at nk = 1 and the view reindexed to 0);
      negC   the negation of such a view of the negated rows: the lanes are a view, the weights a new array;
      reidx  reindex to nk of a batch built with another key split."""
    cols, w = data
    if kind == "fresh":
        return be.batch_from_sorted(s, cols, w, len(w), False)
    if kind == "reidx":
        other = s.reindex((s.nk + 1) % (s.nl + 1))
        return be.reindex(be.batch_from_sorted(other, cols, w, len(w), False), s.nk)
    neg, c = kind.startswith("neg"), int(kind[-1])
    s1 = s if s.nk else s.reindex(1)
    full = concat(s, cut_rows(s, c), (cols, negw(w) if neg else w))
    b = be.batch_from_sorted(s1, full[0], full[1], len(full[1]), False)
    v = be.truncate_keys_below(b, [TMIN[s1.key[0]] + c] + [TMIN[t] for t in s1.key[1:]])
    if s1 != s:
        v = be.reindex(v, s.nk)
    return be.neg(v) if neg else v


def dests(s, cols, P):
    n = len(cols[0]) if cols else 0
    return xm.dests(cols[: s.nk], P) if s.nk and n else np.zeros(n, np.int64)


def shard_view(be, s, data, P, p):
    """Shard p of shard_partition(data, P) (a view into one buffer holding all P shards), and its model rows."""
    parts = be.shard_partition(view(be, s, data, "fresh"), P)
    return parts[p], select(data, dests(s, data[0], P) == p)


# ---- from_tuples ---------------------------------------------------------------------
def raw_rows(rng, s, n, mode):
    """Unsorted rows with duplicates, for from_tuples."""
    cols = [lane_values(rng, s, l, n, mode) for l in range(s.nl)]
    cols, w = ec.with_duplicates(rng, cols, small_weights(rng, n))
    p = rng.permutation(n)
    return [c[p] for c in cols], w[p]


def run_from_tuples(be, ref, s):
    rng = np.random.default_rng(seed_of("from_tuples", s))
    for n in sizes(s.nl):
        for mode in modes_at(s, n):
            cols, w = raw_rows(rng, s, n, mode)
            check(be, ref, lambda b: b.batch_from_columns(s, cols, w), em.consolidate_np(s, cols, w),
                  f"from_tuples {sid(s)} n={n} {mode}")


def device_columns(b, cols, w, offsets, w_offset, alias):
    """torch columns (on the GPU for the CUDA backend, on the CPU for the oracle), lane l starting offsets[l]
    elements into its own buffer; alias = (l, j): lane j passes lane l's tensor itself."""
    import torch

    dev = "cuda" if b.name == "cuda" else "cpu"

    def place(x, o):
        buf = torch.zeros(len(x) + 4, dtype=torch.int64, device=dev)
        buf[o:o + len(x)] = torch.from_numpy(np.ascontiguousarray(x).view(np.int64)).to(dev)
        return buf[o:o + len(x)]

    ts = [place(c, o) for c, o in zip(cols, offsets)]
    if alias is not None:
        ts[alias[1]] = ts[alias[0]]
    return ts, place(w, w_offset)


def run_from_device(be, ref, s):
    """dbsp_batch_from_tuples(on_device=1) reads the caller's columns in place: every lane at its own element
    offset 0..3 (so at its own 16-byte phase), the weights at another; at >= 2 lanes also one tensor passed for
    two lanes (the packing plan's aliased lane)."""
    rng = np.random.default_rng(seed_of("from_device", s))
    T = tile(s.nl)
    for n in (1, T + 1, 3 * T + 2, BIG):
        for mode in modes_at(s, n):
            cols, w = raw_rows(rng, s, n, mode)
            offs = [(l + n) % 4 for l in range(s.nl)]
            aliases = [None] + ([(0, s.nl - 1)] if s.nl >= 2 and n < BIG else [])
            for alias in aliases:
                mc = list(cols)
                if alias is not None:
                    mc[alias[1]] = mc[alias[0]]
                exp = em.consolidate_np(s, mc, w)
                check(be, ref, lambda b: b.batch_from_device_tensors(s, *device_columns(b, cols, w, offs, 3 - n % 4,
                                                                                       alias)),
                      exp, f"from device columns {sid(s)} n={n} {mode} alias={alias}")


# ---- merge ---------------------------------------------------------------------------
MERGE_VIEWS = [("fresh", "fresh"), ("fresh", "cut1"), ("cut1", "cut2"), ("cut3", "cut1"), ("neg1", "fresh"),
               ("cut2", "neg3"), ("neg1", "neg2"), ("reidx", "cut3")]


def merge_pair(rng, s, n, mode):
    """(a, b) consolidated, n rows in all; about 40 % of b's rows repeat a's rows, 70 % of those with the negated
    weight (the pair cancels), the others with weight 1."""
    na, nb = (n + 1) // 2, n // 2
    a = rows(rng, s, na, mode)
    bc, bw = rows(rng, s, nb, mode)
    if na and nb:
        hit = np.flatnonzero(rng.random(nb) < 0.4)
        src = np.sort(rng.choice(na, min(len(hit), na), replace=False))
        hit = hit[: len(src)]
        for c, ac in zip(bc, a[0]):
            c[hit] = ac[src]
        bw[hit] = np.where(rng.random(len(hit)) < 0.7, negw(a[1][src]), 1)
    b = em.consolidate_np(s, bc, bw)
    return a, b


def merged(s, a, b, vb=None):
    cols, w = em.consolidate_np(s, *concat(s, a, b))
    if vb is not None and s.nv:
        cols, w = select((cols, w), ge_lex(cols[s.nk:], s.val, vb))
    return cols, w


def value_bound(s, data):
    """The value lanes of a row about a third into the data (or the types' minima)."""
    cols, w = data
    if not len(w):
        return [TMIN[t] for t in s.val]
    i = len(w) // 3
    return [em.typed(t, int(c[i])) for t, c in zip(s.val, cols[s.nk:])]


def run_merge(be, ref, s):
    rng = np.random.default_rng(seed_of("merge", s))
    for i, n in enumerate(sizes(s.nl)):
        mode = MODES[i % 3]
        a, b = merge_pair(rng, s, n, mode)
        pairs = MERGE_VIEWS if n < BIG else MERGE_VIEWS[2:4] + MERGE_VIEWS[5:6]
        for va, vb_ in pairs:
            check(be, ref, lambda x: x.merge(view(x, s, a, va), view(x, s, b, vb_)), merged(s, a, b),
                  f"merge {sid(s)} n={n} {mode} {va}+{vb_}")
        if s.nv:
            bound = value_bound(s, a)
            check(be, ref, lambda x: x.merge(view(x, s, a, "cut1"), view(x, s, b, "neg2"), val_lower_bound=bound),
                  merged(s, a, b, bound), f"merge_bounded {sid(s)} n={n} {mode}")
        if n >= 3:   # shards of one batch merged with shards of another (views at unrelated offsets)
            sa, ma = shard_view(be, s, a, 3, 1)
            sb, mb = shard_view(be, s, b, 3, 1 if s.nk else 0)
            exp = merged(s, ma, mb)
            got = be.merge(sa, sb)
            em.assert_batch_is(got, exp, f"merge of shards {sid(s)} n={n}")
            if ref is not None:
                assert_batches_equal(got, ref.merge(shard_view(ref, s, a, 3, 1)[0],
                                                    shard_view(ref, s, b, 3, 1 if s.nk else 0)[0]),
                                     f"merge of shards {sid(s)} n={n}: vs {ref.name}")


def run_merger(be, ref, s):
    """The fuelled merger over sliced inputs: every call cuts both inputs at a merge-path split (k_merge_split<L>),
    merges the two slices and appends the chunk."""
    rng = np.random.default_rng(seed_of("merger", s))
    T = tile(s.nl)
    for i, n in enumerate(sizes(s.nl)[1:]):
        mode = MODES[i % 3]
        a, b = merge_pair(rng, s, n, mode)
        va, vb_ = MERGE_VIEWS[2 + i % 6]
        for fuel in (1, 7, T - 1, T + 1, 1 << 40):
            if (fuel == 1 and n > T + 1) or (fuel == 7 and n > 3 * T + 2):
                continue
            bound = value_bound(s, a) if s.nv and fuel == 7 else None

            def fuelled(x):
                m = x.merger(view(x, s, a, va), view(x, s, b, vb_), val_lower_bound=bound)
                while m.work(fuel) <= 0:
                    pass
                return m.done()

            check(be, ref, fuelled, merged(s, a, b, bound), f"merger {sid(s)} n={n} {mode} {va}+{vb_} fuel={fuel}")


# ---- spine ---------------------------------------------------------------------------
def run_spine(be, ref, s):
    """Inserts of fresh and sliced batches, then truncate_keys_below, truncate_values_below, exert, consolidate."""
    rng = np.random.default_rng(seed_of("spine", s))
    T = tile(s.nl)
    for n, mode in ((T + 1, "narrow"), (3 * T + 2, "mixed"), (3 * T + 2, "full")):
        parts = [rows(rng, s, m, mode) for m in (n, n // 2, n // 3, n // 5)]
        kinds = ("fresh", "cut1", "neg3", "cut2")
        allr = em.consolidate_np(s, *concat(s, *parts))
        kb = [em.typed(t, int(c[len(allr[1]) // 4])) for t, c in zip(s.key, allr[0][: s.nk])] if s.nk else []
        exp = select(allr, ge_lex(allr[0][: s.nk], s.key, kb)) if s.nk else allr
        vb = value_bound(s, exp) if s.nv else None
        if vb is not None:
            exp = select(exp, ge_lex(exp[0][s.nk:], s.val, vb))

        def op(x):
            sp = Spine(x, s)
            for p, k in zip(parts, kinds):
                sp.insert(view(x, s, p, k))
            if s.nk:
                sp.truncate_keys_below(kb)
            if vb is not None:
                sp.truncate_values_below(vb)
            sp.exert(n)
            return sp.consolidate()

        check(be, ref, op, exp, f"spine {sid(s)} n={n} {mode}")


# ---- reindex, key count, CSR download -------------------------------------------------
def run_reindex(be, ref, s):
    rng = np.random.default_rng(seed_of("reindex", s))
    T = tile(s.nl)
    for n, mode in ((1, "narrow"), (T + 1, "narrow"), (3 * T + 2, "mixed"), (BIG, modes_at(s, BIG)[0])):
        data = rows(rng, s, n, mode)
        for kind in ("fresh", "cut3") if n < BIG else ("cut3",):
            for nk in range(s.nl + 1):
                s2 = s.reindex(nk)
                what = f"reindex {sid(s)} -> {nk} n={n} {mode} {kind}"
                got = check(be, ref, lambda x: x.reindex(view(x, s, data, kind), nk), data, what)
                assert got.schema == s2
                head = np.ones(n, bool)   # rows whose first nk lanes differ from the previous row's
                head[1:] = False
                for c in data[0][:nk]:
                    head[1:] |= c[1:] != c[:-1]
                assert got.key_count() == (n if not s2.nv else int(head.sum())), what
                if nk == 0 and s2.nv:
                    d = got.download()
                    assert d["keys"] == [] and list(d["offs"]) == ([0, n] if n else [0]), what


# ---- join, semijoin ------------------------------------------------------------------
def join_proj(s, rs, swap=False):
    """Up to 8 output lanes: the key lanes, then the left and the right value lanes."""
    ls = rs if swap else s
    other = s if swap else rs
    srcs = [(key(i), s.key[i]) for i in range(s.nk)] + [(lval(j), ls.val[j]) for j in range(ls.nv)]
    srcs += [(rval(j), other.val[j]) for j in range(other.nv)]
    srcs = srcs[:8]
    types = "".join(t for _, t in srcs)
    onk = min(max(s.nk, 1), len(srcs))
    return Proj(Schema(types[:onk], types[onk:]), [e for e, _ in srcs])


def right_side(rng, s, left, n):
    """Rows of schema Schema(s.key, 2 value lanes or fewer) whose keys are drawn from the left rows' keys."""
    rs = Schema(s.key, ("ui" * 4)[: min(2, 8 - s.nk)])
    if not len(left[1]):
        return rs, rows(rng, rs, 0, "narrow")
    pick = rng.integers(0, len(left[1]), n)
    cols = [c[pick] for c in left[0][: s.nk]] + [lane_values(rng, rs, s.nk + j, n, "narrow") for j in range(rs.nv)]
    return rs, em.consolidate_np(rs, cols, small_weights(rng, n))


def join_sizes(s):
    return (1, 120) if s.nk == 0 else (1, 300, 900)


def run_join(be, ref, s):
    rng = np.random.default_rng(seed_of("join", s))
    bes = [be] + ([ref] if ref is not None else [])
    for i, n in enumerate(join_sizes(s)):
        left = rows(rng, s, n, MODES[i % 3] if s.nk else "narrow")
        rs, right = right_side(rng, s, left, max(1, (2 * n) // 3))
        zl, zr = z_of(s, left), z_of(rs, right)
        proj = join_proj(s, rs)
        for kl, kr in (("fresh", "fresh"), ("cut1", "neg2"), ("neg3", "cut1")):
            check(be, ref, lambda x: x.join_batches(view(x, s, left, kl), view(x, rs, right, kr), proj),
                  em.join(zl, zr, proj), f"join_batches {sid(s)} n={n} {kl}x{kr}")
        # join_delta_trace: the right rows split over a trace of three batches, two of them views
        thirds = [select(right, np.arange(len(right[1])) % 3 == r) for r in range(3)]
        spines = [Spine(x, rs) for x in bes]
        for sp, x in zip(spines, bes):
            for part, k in zip(thirds, ("cut1", "fresh", "neg3")):
                sp.insert(view(x, rs, part, k))
        for left_is_delta in (True, False):
            p = proj if left_is_delta else join_proj(s, rs, swap=True)
            exp = em.join_delta_trace(zl, zr, p, delta_is_left=left_is_delta)
            what = f"join_delta_trace {sid(s)} n={n} delta_is_left={left_is_delta}"
            got = be.join_delta_trace(view(be, s, left, "cut3"), spines[0], p, delta_is_left=left_is_delta)
            em.assert_batch_is(got, exp, what)
            if ref is not None:
                assert_batches_equal(got, ref.join_delta_trace(view(ref, s, left, "cut3"), spines[1], p,
                                                               delta_is_left=left_is_delta), f"{what}: vs {ref.name}")


def run_traces(be, ref, s):
    """semijoin (nk >= 1), distinct_delta and Max / Min aggregates over traces of several batches, some of them
    slices."""
    rng = np.random.default_rng(seed_of("traces", s))
    bes = [be] + ([ref] if ref is not None else [])
    ks = Schema(s.key)
    for i, n in enumerate((1, 200, 1200)):
        mode = MODES[i % 3]
        data = rows(rng, s, n, mode)
        if s.nk:
            pick = rng.integers(0, n, max(1, n // 2))
            kcols, kw = em.consolidate_np(ks, [c[pick] for c in data[0][: s.nk]], ec.edge_weights(rng, len(pick)))
            check(be, ref, lambda x: x.semijoin(view(x, s, data, "cut1"), view(x, ks, (kcols, kw), "neg3")),
                  em.semijoin(z_of(s, data), z_of(ks, (kcols, kw))), f"semijoin {sid(s)} n={n}")
        # distinct: the integral in three batches, a delta that repeats some of its rows
        parts = [select(data, np.arange(n) % 3 == r) for r in range(3)]
        dl = rows(rng, s, max(1, n // 3), mode)
        back = select(data, np.arange(n) % 4 == 0)
        delta = em.consolidate_np(s, *concat(s, dl, (back[0], negw(back[1]))))

        def op(x):
            sp = Spine(x, s)
            for p, k in zip(parts, ("fresh", "cut1", "neg2")):
                sp.insert(view(x, s, p, k))
            return x.distinct_delta(view(x, s, delta, "cut3"), sp)

        check(be, ref, op, em.distinct_delta(z_of(s, delta), z_of(s, data)), f"distinct_delta {sid(s)} n={n}")
        if not s.nv:
            continue
        for kind in (capi.AGG_MAX, capi.AGG_MIN):
            ins, outs = [Spine(x, s) for x in bes], [Spine(x, s) for x in bes]
            zin, zout = Z(s), Z(s)
            steps = [(parts[0], "cut1"), (parts[1], "neg3"), (parts[2], "fresh"),
                     (em.consolidate_np(s, data[0], negw(data[1])), "cut2")]
            for j, (d, k) in enumerate(steps):
                zd = z_of(s, d)
                zin.add(zd.rows())
                exp = em.aggregate_delta(zd, zin, zout, kind)
                res = []
                for sp, osp, x in zip(ins, outs, bes):
                    b = view(x, s, d, k)
                    sp.insert(b)
                    res.append(x.aggregate_delta(b, sp, osp, kind))
                    osp.insert(res[-1])
                what = f"aggregate {'max' if kind == capi.AGG_MAX else 'min'} {sid(s)} n={n} step {j}"
                em.assert_batch_is(res[0], exp, what)
                if ref is not None:
                    assert_batches_equal(res[0], res[1], f"{what}: vs {ref.name}")
                zout.add(exp.rows())


# ---- shard_partition -----------------------------------------------------------------
def run_shards(be, ref, s):
    """Every shard equals the model's rows for it (exchange_model's placement; at nk = 0 every row goes to shard
    0), also when the input is a view."""
    rng = np.random.default_rng(seed_of("shards", s))
    T = tile(s.nl)
    for n, mode in ((1, "narrow"), (T + 1, "mixed"), (3 * T + 2, "full"), (BIG, modes_at(s, BIG)[0])):
        data = rows(rng, s, n, mode)
        for kind in ("fresh", "cut1", "neg3", "reidx") if n < BIG else ("cut1",):
            for P in (1, 2, 3, 7):
                d = dests(s, data[0], P)
                if not s.nk:
                    assert not d.any()
                parts = be.shard_partition(view(be, s, data, kind), P)
                rparts = ref.shard_partition(view(ref, s, data, kind), P) if ref is not None else [None] * P
                for p, (got, other) in enumerate(zip(parts, rparts)):
                    what = f"shard {p} of {P} {sid(s)} n={n} {mode} {kind}"
                    em.assert_batch_is(got, select(data, d == p), what)
                    if other is not None:
                        assert_batches_equal(got, other, f"{what}: vs {ref.name}")


# ---- window --------------------------------------------------------------------------
def run_window(be, ref, s):
    """Window retractions are negated slices of the trace's batches (their own weights, lanes at the slice's
    offset) merged by a merge tree; at 1 and 2 lanes a slice at an odd offset makes the merge stage with cp.async.
    Two trace batches (keys 10j and 10j + 5) of several tiles each; the windows move so that the retracted regions
    start at odd and even offsets and span several tiles."""
    T = tile(s.nl)
    rng = np.random.default_rng(seed_of("window", s))
    kt = s.key[0]
    k = lambda j: TMIN[kt] + 10 * j

    def batch_rows(n, off):
        cols = [np.array([em.u64(k(j) + off) for j in range(n)], np.uint64)]
        cols += [lane_values(rng, s, l, n, "narrow") for l in range(1, s.nl)]
        return em.consolidate_np(s, cols, small_weights(rng, n))

    parts = [batch_rows(6 * T, 0), batch_rows(3 * T, 5)]
    trace = z_of(s, concat(s, *parts))
    drows = batch_rows(5 * T, 3)
    delta = z_of(s, drows)
    wins = [None, (k(1), k(4 * T + 1)), (k(2 * T + 3), k(5 * T)), (k(3 * T + 1), k(3 * T + 2)),
            (k(3 * T + 1), k(6 * T))]
    for prev, cur in zip(wins, wins[1:]):
        pb = None if prev is None else ([prev[0]], [prev[1]])
        exp = em.window_delta(trace, delta, pb, ([cur[0]], [cur[1]]))

        def win(x):
            sp = Spine(x, s)
            for p, kind in zip(parts, ("fresh", "cut1")):
                sp.insert(view(x, s, p, kind))
            return x.window_delta(sp, view(x, s, drows, "cut3"), pb, ([cur[0]], [cur[1]]))

        check(be, ref, win, exp, f"window {sid(s)} {prev} -> {cur}")


WINDOW_SHAPES = [Schema("u"), Schema("i"), Schema("u", "i"), Schema("i", "u")]

PER_SHAPE = {"from_tuples": run_from_tuples, "from_device": run_from_device, "merge": run_merge,
             "merger": run_merger, "spine": run_spine, "reindex": run_reindex, "join": run_join,
             "traces": run_traces, "shards": run_shards}
ALL_CASES = {}
for _op, _fn in PER_SHAPE.items():
    for _s in SHAPES:
        ALL_CASES[f"{_op}_L{_s.nl}_{sid(_s)}"] = lambda be, ref=None, fn=_fn, s=_s: fn(be, ref, s)
for _s in WINDOW_SHAPES:
    ALL_CASES[f"window_L{_s.nl}_{sid(_s)}"] = lambda be, ref=None, s=_s: run_window(be, ref, s)

# the cases that merge (the subset run again with DBSP_MERGE_NO_TMA=1), grouped by merge configuration
NO_TMA_OPS = ("merge", "merger", "spine", "window")
NO_TMA_GROUPS = {"L1-2": (1, 2), "L3-6": (3, 4, 5, 6), "L7-8": (7, 8)}


def no_tma_cases(group):
    lanes = NO_TMA_GROUPS[group]
    return sorted(n for n in ALL_CASES if n.split("_L")[0] in NO_TMA_OPS and int(n.split("_L")[1].split("_")[0]) in lanes)


if __name__ == "__main__":
    # python tests/shape_cases.py GROUP: the NO_TMA subset of one group on CUDA, against the model and the oracle
    import dbsp_b200.runtime as rt
    from oracle_backend import OracleBackend

    group = sys.argv[1]
    assert os.environ.get("DBSP_MERGE_NO_TMA"), "run with DBSP_MERGE_NO_TMA=1"
    cuda, oracle = rt.Runtime(0), OracleBackend()
    names = no_tma_cases(group)
    for name in names:
        ALL_CASES[name](cuda, oracle)
    print(f"SHAPES_OK {group} {len(names)} cases", flush=True)
