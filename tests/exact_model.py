"""An exact model of the row language and the operators of include/dbsp_b200.h, in plain Python ints with
explicit two's complement (DESIGN §2): lanes are u64 or i64, weights wrap mod 2^64, a row whose summed weight is 0
does not exist.  It shares no code with the oracle or the library; only the `Src` / `Expr` / `Pred` / `Proj`
objects the tests build are read.

A Z-set is a `Z`: a schema and a dict {row tuple: weight}, every lane held as its typed value (`u` lanes in
[0, 2^64), `i` lanes in [-2^63, 2^63)), so Python's tuple order is the lanes' order.  Large consolidations and
merges go through `consolidate_np`, a numpy uint64 path with the same rules."""
import numpy as np

from dbsp_b200 import capi

M64 = 1 << 64
MIN, MAX = -(1 << 63), (1 << 63) - 1
UMAX = M64 - 1
SIGN = np.uint64(1 << 63)


def w64(x):
    """x reduced mod 2^64 into [-2^63, 2^63)."""
    x &= UMAX
    return x - M64 if x >> 63 else x


def u64(x):
    return x & UMAX


def typed(t, x):
    return w64(x) if t == "i" else u64(x)


class Z:
    def __init__(self, schema, rows=None):
        self.schema, self.d = schema, {}
        if rows is not None:
            self.add(rows)

    def add(self, rows, sign=1):
        """rows: (lane.., weight) tuples; lanes are reduced to their types, weights summed mod 2^64."""
        ts = self.schema.lanes
        for r in rows:
            t = tuple(typed(ty, x) for ty, x in zip(ts, r[:-1]))
            w = w64(self.d.get(t, 0) + sign * r[-1])
            if w:
                self.d[t] = w
            else:
                self.d.pop(t, None)
        return self

    def rows(self):
        return [t + (w,) for t, w in sorted(self.d.items())]

    def copy(self):
        z = Z(self.schema)
        z.d = dict(self.d)
        return z

    def groups(self):
        """{key: [(val, weight), ..] in value order}"""
        nk, g = self.schema.nk, {}
        for t, w in sorted(self.d.items()):
            g.setdefault(t[:nk], []).append((t[nk:], w))
        return g


def groups_of(z, keys):
    """Z.groups() restricted to `keys`."""
    nk, ks, g = z.schema.nk, set(keys), {}
    for t, w in sorted((t, w) for t, w in z.d.items() if t[:z.schema.nk] in ks):
        g.setdefault(t[:nk], []).append((t[nk:], w))
    return g


def union(*zs):
    out = Z(zs[0].schema)
    for z in zs:
        out.add(z.rows())
    return out


def neg(z):
    return Z(z.schema, [r[:-1] + (-r[-1],) for r in z.rows()])


# ---- the row language ------------------------------------------------------------
def src(s, env):
    """A source's u64 bit pattern.  env = (key lanes, lval lanes, rval lanes), each a tuple of typed ints."""
    if s.kind == capi.SRC_CONST:
        return u64(s.cst)
    part = {capi.SRC_KEY: 0, capi.SRC_LVAL: 1, capi.SRC_RVAL: 2}[s.kind]
    return u64(env[part][s.idx])


def expr(e, env):
    """u64 bit pattern of an Expr: wrapping NEG/ADD/SUB/MUL; DIV = i64::wrapping_div with x / 0 = 0."""
    a = src(e.a, env)
    if e.op == capi.OP_COPY:
        return a
    if e.op == capi.OP_NEG:
        return u64(-a)
    b = src(e.b, env)
    if e.op == capi.OP_ADD:
        return u64(a + b)
    if e.op == capi.OP_SUB:
        return u64(a - b)
    if e.op == capi.OP_MUL:
        return u64(a * b)
    assert e.op == capi.OP_DIV, e.op
    sa, sb = w64(a), w64(b)
    if sb == 0:
        return 0
    q = abs(sa) // abs(sb)   # truncation toward zero
    return u64(q if (sa < 0) == (sb < 0) else -q)


def pred(p, env):
    a, b = src(p.a, env), src(p.b, env)
    if p.cmp == capi.CMP_IN:
        return a < 64 and (b >> a) & 1 == 1
    if p.is_signed:
        a, b = w64(a), w64(b)
    return {capi.CMP_EQ: a == b, capi.CMP_NE: a != b, capi.CMP_LT: a < b, capi.CMP_LE: a <= b,
            capi.CMP_GT: a > b, capi.CMP_GE: a >= b}[p.cmp]


def project(proj, env):
    """The output row (typed lanes) or None when a predicate fails."""
    if not all(pred(p, env) for p in proj.where):
        return None
    return tuple(typed(t, expr(e, env)) for t, e in zip(proj.schema.lanes, proj.out))


# ---- batch operators -------------------------------------------------------------
def merge_bounded(a, b, vb):
    """Union with the values below `vb` dropped (keys left without values vanish); OrdZSets ignore the bound."""
    out = union(a, b)
    s = out.schema
    if vb is None or s.nv == 0:
        return out
    bound = tuple(typed(t, x) for t, x in zip(s.val, vb))
    out.d = {t: w for t, w in out.d.items() if t[s.nk:] >= bound}
    return out


def map_index(z, proj):
    out = Z(proj.schema)
    nk = z.schema.nk
    for t, w in z.d.items():
        r = project(proj, (t[:nk], t[nk:], t[nk:]))
        if r is not None:
            out.add([r + (w,)])
    return out


def batch_from_table(cols, proj, weights=None):
    """flat_map_index over a raw table: key(i), lval(i) and rval(i) all read column i."""
    out = Z(proj.schema)
    n = len(cols[0])
    cl = [[int(x) for x in np.asarray(c).view(np.uint64)] for c in cols]
    for i in range(n):
        row = tuple(c[i] for c in cl)
        r = project(proj, (row, row, row))
        if r is not None:
            out.add([r + (1 if weights is None else int(weights[i]),)])
    return out


def join(left, right, proj, swap=False):
    """Join::eval: on equal keys every (v1, v2) pair, weight w1*w2 mod 2^64.  swap: `right` feeds lval."""
    out = Z(proj.schema)
    gr = right.groups()
    for k, lvs in left.groups().items():
        for v1, w1 in lvs:
            for v2, w2 in gr.get(k, ()):
                env = (k, v2, v1) if swap else (k, v1, v2)
                r = project(proj, env)
                if r is not None:
                    out.add([r + (w1 * w2,)])
    return out


def join_delta_trace(delta, trace, proj, delta_is_left=True):
    return join(delta, trace, proj, swap=not delta_is_left)


def semijoin(pairs, keys):
    from dbsp_b200 import Schema

    out = Z(Schema(pairs.schema.lanes))
    nk = pairs.schema.nk
    for t, w in pairs.d.items():
        kw = keys.d.get(t[:nk], 0)
        if kw:
            out.add([t + (w * kw,)])
    return out


def weigh(z, f, mode):
    """LINEAR: (k) -> sum f(k,v)*w.  AVG: (k,0) -> sum f(k,v)*w, (k,1) -> sum w."""
    from dbsp_b200 import Schema

    avg = mode == capi.WEIGH_AVG
    out = Z(Schema(z.schema.key + ("u" if avg else "")))
    for k, vs in z.groups().items():
        s = sum(expr(f, (k, v, v)) * w for v, w in vs)
        c = sum(w for v, w in vs)
        if avg:
            out.add([k + (0, s), k + (1, c)])
        else:
            out.add([k + (s,)])
    return out


def aggregate_value(kind, vals, out_schema):
    """f(integral) of one key: vals = [(val, weight != 0)] in value order; None = no output row."""
    if kind == capi.AGG_MAX:
        return vals[-1][0] if vals else None
    if kind == capi.AGG_MIN:
        return vals[0][0] if vals else None
    if kind == capi.AGG_FOLD_COUNT:
        return (len(vals),) if vals else None
    if kind == capi.AGG_FOLD_SUM:
        return (u64(sum(u64(v[0]) for v, _ in vals)),) if vals else None
    if kind == capi.AGG_WCOUNT:
        s = w64(sum(w for _, w in vals))
        return (s,) if s else None
    raise ValueError(kind)


def aggregate_delta(delta, in_trace, out_trace, kind):
    """AggregateIncremental + Upsert for the keys of `delta`: -old value, +f(in_trace), as consolidated rows.
    in_trace already holds the delta.  WCOUNT2: delta and in_trace are OrdZSet<(K.., which)>; f = (sum, count)."""
    os_ = out_trace.schema
    nk = os_.nk
    out = Z(os_)
    keys = sorted({t[:nk] for t in delta.d})
    g_in, g_out = groups_of(in_trace, keys), groups_of(out_trace, keys)
    for k in keys:
        if kind == capi.AGG_WCOUNT2:
            s, c = (w64(in_trace.d.get(k + (wh,), 0)) for wh in (0, 1))
            new = (s, c) if (s or c) else None
        else:
            new = aggregate_value(kind, g_in.get(k, []), os_)
        rows = [k + v + (-w,) for v, w in g_out.get(k, [])]
        if new is not None:
            rows.append(k + tuple(typed(t, x) for t, x in zip(os_.val, new)) + (1,))
        out.add(rows)
    return out


def distinct_delta(delta, integral):
    """DistinctIncrementalTotal: old = integral weight, new = old + delta (mod 2^64); +1 when old <= 0 < new,
    -1 when new <= 0 < old."""
    out = Z(delta.schema)
    for t, w in delta.d.items():
        old = integral.d.get(t, 0)
        new = w64(old + w)
        if old <= 0 < new:
            out.add([t + (1,)])
        elif new <= 0 < old:
            out.add([t + (-1,)])
    return out


def stream_distinct(z):
    return Z(z.schema, [t + (1,) for t, w in z.d.items() if w > 0])


def _key(schema, k):
    return tuple(typed(t, x) for t, x in zip(schema.key, k))


def truncate_keys_below(z, bound):
    b = _key(z.schema, bound)
    out = Z(z.schema)
    out.d = {t: w for t, w in z.d.items() if t[: z.schema.nk] >= b}
    return out


def window_delta(trace, delta, prev, cur):
    """Window::eval on the keys: trace rows that left [start0, end0) for [start1, end1) with -w, those that entered
    with +w, plus the delta's rows inside [start1, end1)."""
    s = delta.schema
    nk = s.nk
    s1, e1 = _key(s, cur[0]), _key(s, cur[1])
    out = Z(s)
    inside1 = lambda k: s1 <= k < e1
    for t, w in delta.d.items():
        if inside1(t[:nk]):
            out.add([t + (w,)])
    if prev is not None:
        s0, e0 = _key(s, prev[0]), _key(s, prev[1])
        for t, w in trace.d.items():
            k = t[:nk]
            was, now = s0 <= k < e0, inside1(k)
            if was and not now:
                out.add([t + (-w,)])
            elif now and not was:
                out.add([t + (w,)])
    return out


def last_key(z):
    return max(t[: z.schema.nk] for t in z.d) if z.d else None


# ---- backend batches <-> model ---------------------------------------------------
def of_batch(b):
    """The Z of a backend batch (small and medium batches)."""
    return Z(b.schema, b.rows())


def flat(schema, z):
    """Sorted flat rows as numpy columns (uint64 bit patterns) and int64 weights."""
    rows = z.rows()
    cols = [np.array([u64(r[l]) for r in rows], dtype=np.uint64) for l in range(schema.nl)]
    return cols, np.array([r[-1] for r in rows], dtype=np.int64)


def flips(schema):
    return [SIGN if t == "i" else np.uint64(0) for t in schema.lanes]


def lex_order(keyed):
    """np.lexsort(keyed[::-1]) (stable, lane 0 most significant) for uint64 lanes, by np.sort alone: every lane's
    offset from its minimum takes its bit width, the lanes are concatenated (the last lane least significant) and
    the concatenation is sorted in digits of 64 - ib bits, least significant digit first, each digit with the
    row's current position in the low ib bits (distinct words: np.sort is then a stable sort by the digit).
    Returns (order, the digits of every pass in that order: equal rows have equal digits)."""
    n = len(keyed[0])
    ib = max((n - 1).bit_length(), 1)
    dbits = 64 - ib
    offs, bits = [], []
    for c in keyed:
        mn = c.min()
        offs.append(c - mn)
        bits.append(int(c.max() - mn).bit_length())
    total, pos, at = sum(bits), [0] * len(keyed), 0
    for l in range(len(keyed) - 1, -1, -1):
        pos[l], at = at, at + bits[l]
    low, sh = np.uint64((1 << ib) - 1), np.uint64(ib)
    order, digits = None, []
    for lo in range(0, max(total, 1), dbits):
        hi = min(lo + dbits, total)
        d = np.zeros(n, np.uint64)
        for o, p, b in zip(offs, pos, bits):   # bits [lo, hi) of the concatenation
            if b and p < hi and p + b > lo:
                d |= (o >> np.uint64(max(lo - p, 0))) << np.uint64(max(p - lo, 0))
        if hi > lo:
            d &= np.uint64((1 << (hi - lo)) - 1)
        s = np.sort(((d if order is None else d[order]) << sh) | np.arange(n, dtype=np.uint64))
        perm = (s & low).astype(np.int64)
        order = perm if order is None else order[perm]
        digits.append(d)
    # the last pass's digit comes out of the sort in order; the earlier ones are gathered
    return order, [d[order] for d in digits[:-1]] + [s >> sh]


def consolidate_np(schema, cols, weights):
    """from_tuples on numpy uint64 columns: sort by the typed lanes, sum equal rows mod 2^64, drop zero sums.
    Returns (sorted cols, weights)."""
    n = len(weights)
    if n == 0:
        return [np.zeros(0, np.uint64) for _ in range(schema.nl)], np.zeros(0, np.int64)
    cols = [np.asarray(c).view(np.uint64) for c in cols]
    keyed = [c ^ f for c, f in zip(cols, flips(schema))]
    order, digits = lex_order(keyed) if keyed else (np.arange(n), [])
    w = np.asarray(weights).view(np.uint64)[order]
    head = np.ones(n, bool)
    head[1:] = False
    for d in digits:   # the packing is injective: rows differ iff some digit differs
        head[1:] |= d[1:] != d[:-1]
    starts = np.flatnonzero(head)
    sums = np.add.reduceat(w, starts)   # uint64: wraps mod 2^64 by definition
    keep = sums != 0
    rows = order[starts[keep]]
    return [c[rows] for c in cols], sums[keep].view(np.int64)


def canon(schema, cols, weights):
    """The canonical keys / offs / vals / diffs vectors of sorted, consolidated flat rows."""
    nk = schema.nk
    n = len(weights)
    if schema.nv == 0:
        keys, offs, vals = cols, None, []
    else:
        head = np.ones(n, bool)
        if n:
            head[1:] = False
            for c in cols[:nk]:
                head[1:] |= c[1:] != c[:-1]
        starts = np.flatnonzero(head)
        keys = [c[starts] for c in cols[:nk]]
        offs = np.append(starts, n).astype(np.uint64)
        vals = cols[nk:]
    view = lambda t, c: c.view(np.int64) if t == "i" else c
    return {"keys": [view(t, c) for t, c in zip(schema.key, keys)], "offs": offs,
            "vals": [view(t, c) for t, c in zip(schema.val, vals)], "diffs": np.asarray(weights, np.int64)}


def assert_batch_is(b, expect, what=""):
    """Backend batch `b` == the model's result: a Z, or (cols, weights) from consolidate_np."""
    if isinstance(expect, Z):
        assert b.schema == expect.schema, f"{what}: schema {b.schema} != {expect.schema}"
    assert_download_is(b.schema, b.download(), expect, what)


def assert_download_is(schema, got, expect, what=""):
    """A batch of `schema` already downloaded (Batch.download()) == the model's result: a Z, or (cols, weights)
    from consolidate_np."""
    if isinstance(expect, Z):
        cols, w = flat(schema, expect)
    else:
        cols, w = expect
    want = canon(schema, cols, w)
    assert len(got["diffs"]) == len(want["diffs"]), f"{what}: {len(got['diffs'])} tuples, model has {len(want['diffs'])}"
    for part in ("keys", "vals"):   # a download missing a lane must not pass by zip's truncation
        assert len(got[part]) == len(want[part]), f"{what}: {len(got[part])} {part} lanes, model has {len(want[part])}"
    for part in ("keys", "vals"):
        for i, (x, y) in enumerate(zip(got[part], want[part])):
            assert np.array_equal(x, y), f"{what}: {part} lane {i} differs from the model"
    if want["offs"] is not None:
        assert np.array_equal(got["offs"], want["offs"]), f"{what}: offs differ from the model"
    assert np.array_equal(got["diffs"], want["diffs"]), f"{what}: weights differ from the model"
