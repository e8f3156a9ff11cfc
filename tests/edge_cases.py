"""Backend-generic tests at the edges of the integer domain (DESIGN §2): full-range u64 / i64 lanes, weights that
sum to 0 only mod 2^64, products that overflow, the i64 order flip at MIN / MAX, division overflow.  Every case
compares the backend's output with the exact model of tests/exact_model.py; given a second backend (`ref`, the
oracle when the CUDA library is under test) it also compares the two bit for bit."""
import numpy as np

import exact_model as em
from dbsp_b200 import Proj, RootCircuit, Schema, Spine, capi, const, key, lval, rval
from dbsp_b200.zset import Pred
from exact_model import MAX, MIN, UMAX, Z
from parity_util import assert_batches_equal

U_POOL = [0, 1, (1 << 63) - 1, 1 << 63, (1 << 63) + 1, UMAX - 1, UMAX]
I_POOL = [MIN, MIN + 1, -1, 0, 1, MAX - 1, MAX]
W_POOL = [MIN, MIN + 1, 1 << 62, -(1 << 62), 1 << 32, -(1 << 32), 1, -1, MAX]
SCHEMAS = [Schema("u"), Schema("u", "u"), Schema("i", "u"), Schema("uu", "i"), Schema("u", "uuu"), Schema("uu", "uuu"),
           Schema("uiu", "uiuu"), Schema("uuuu", "uuuu"), Schema("i"), Schema("i", "i"), Schema("ii", "iii")]
# runs of equal rows: the first four sum to 0 only mod 2^64; the others wrap to a total whose low 32 bits are 0
WRAP_RUNS = [[1 << 62] * 4, [MAX, MAX, 2], [MIN, MIN], [MIN + 1, MAX], [1 << 62] * 3, [MAX, 1], [1 << 33, -(1 << 32)],
             [1 << 32]]


def sid(s):
    return f"{s.key}_{s.val}"


def check(be, ref, op, expect, what):
    """op(backend) -> batch: equal to the model, and bit-exact with `ref`'s when given."""
    got = op(be)
    em.assert_batch_is(got, expect, what)
    if ref is not None:
        assert_batches_equal(got, op(ref), f"{what}: vs {ref.name}")
    return got


def full_lane(rng, t, n, pool_share=0.3):
    """n values of a full-range lane: random 64-bit patterns with the pool's extremes mixed in (uint64 bits)."""
    x = rng.integers(0, 1 << 64, n, dtype=np.uint64)
    pool = np.array([em.u64(v) for v in (I_POOL if t == "i" else U_POOL)], dtype=np.uint64)
    pick = rng.random(n) < pool_share
    x[pick] = pool[rng.integers(0, len(pool), int(pick.sum()))]
    return x


def edge_weights(rng, n):
    w = rng.integers(MIN, MAX, n, dtype=np.int64, endpoint=True)
    pick = rng.random(n) < 0.6
    w[pick] = np.array(W_POOL, dtype=np.int64)[rng.integers(0, len(W_POOL), int(pick.sum()))]
    return w


def with_duplicates(rng, cols, w):
    """About a third of the rows repeat an earlier row (so equal rows meet in runs)."""
    n = len(w)
    if n > 2:
        d = rng.random(n) < 0.35
        src_rows = rng.integers(0, n, n)
        for c in cols:
            c[d] = c[src_rows[d]]
    return cols, w


def from_cols(be, schema, cols, w):
    return be.batch_from_columns(schema, cols, w)


# ---- consolidation and the sort plans --------------------------------------------
def run_consolidate_full(be, ref, schema, n, seed):
    """Every lane full-range (64 bits wide in the packing plan), extremes, duplicates, edge weights."""
    rng = np.random.default_rng(seed)
    cols, w = with_duplicates(rng, [full_lane(rng, t, n) for t in schema.lanes], edge_weights(rng, n))
    check(be, ref, lambda b: from_cols(b, schema, cols, w), em.consolidate_np(schema, cols, w),
          f"from_tuples full-range {sid(schema)} n={n}")


def run_consolidate_plans(be, ref):
    rng = np.random.default_rng(41)
    n = 70_001
    # exactly 128 bits: two full u64 lanes (0 and 2^64-1 both present), W = 2 with lane 1 at bit 64
    s = Schema("u", "u")
    cols, w = with_duplicates(rng, [full_lane(rng, "u", n), full_lane(rng, "u", n)], edge_weights(rng, n))
    cols[0][:2], cols[1][:2] = np.uint64(0), np.uint64(UMAX)
    cols[0][2:4], cols[1][2:4] = np.uint64(UMAX), np.uint64(0)
    check(be, ref, lambda b: from_cols(b, s, cols, w), em.consolidate_np(s, cols, w), "128-bit key")
    # three and four full lanes: whole lanes per key word, sorted word by word
    for s in (Schema("ui", "u"), Schema("ii", "iu")):
        cols, w = with_duplicates(rng, [full_lane(rng, t, n) for t in s.lanes], edge_weights(rng, n))
        check(be, ref, lambda b: from_cols(b, s, cols, w), em.consolidate_np(s, cols, w), f"word by word {sid(s)}")
    # a presorted lane 0 running from MIN to MAX (the sort-free leading lane), second lane unordered
    s = Schema("i", "u")
    lane0 = np.sort(full_lane(rng, "i", n).view(np.int64))
    lane0[0], lane0[-1] = MIN, MAX
    lane1 = rng.integers(0, 1 << 20, n).astype(np.uint64)
    lane1[::7] = np.uint64(UMAX)
    cols, w = [lane0.view(np.uint64), lane1], edge_weights(rng, n)
    check(be, ref, lambda b: from_cols(b, s, cols, w), em.consolidate_np(s, cols, w), "presorted MIN..MAX lane 0")
    # an aliased lane (equal to lane 0 in every row) holding the extremes
    s = Schema("u", "uu")
    l0 = full_lane(rng, "u", n, pool_share=0.6)
    cols, w = with_duplicates(rng, [l0, full_lane(rng, "u", n), l0.copy()], edge_weights(rng, n))
    cols[2] = cols[0].copy()
    check(be, ref, lambda b: from_cols(b, s, cols, w), em.consolidate_np(s, cols, w), "aliased lane")


def wrap_run_rows(schema, n_rows, shift):
    """Distinct rows in ascending order, each repeated as one of WRAP_RUNS (plus `shift` single rows in front, so
    that runs straddle the 1024-row reduce tiles and the 3072 / 6144-row chunks)."""
    lanes, weights = [], []
    j = 0
    while len(weights) < n_rows:
        run = [1] if j < shift else WRAP_RUNS[j % len(WRAP_RUNS)]
        lanes += [j] * len(run)
        weights += run
        j += 1
    base = np.array(lanes, dtype=np.uint64)
    cols = []
    for l, t in enumerate(schema.lanes):   # monotone in j on every lane; the i lanes sit just above MIN
        c = base * np.uint64(2 * l + 1)
        cols.append((c ^ em.SIGN) if t == "i" else c)
    return cols, np.array(weights, dtype=np.int64)


def run_wrap_runs(be, ref):
    rng = np.random.default_rng(43)
    for s in (Schema("u"), Schema("u", "u"), Schema("i", "u"), Schema("uu", "iuu")):
        for shift in (0, 1, 2):
            cols, w = wrap_run_rows(s, 7000, shift)
            exp = em.consolidate_np(s, cols, w)
            assert len(exp[1]) and not np.any(exp[1] == 0)
            check(be, ref, lambda b: from_cols(b, s, cols, w), exp, f"wrap runs in order {sid(s)} shift={shift}")
            p = rng.permutation(len(w))
            pc, pw = [c[p] for c in cols], w[p]
            check(be, ref, lambda b: from_cols(b, s, pc, pw), exp, f"wrap runs shuffled {sid(s)} shift={shift}")
    # the model's own arithmetic on the runs
    assert [em.w64(sum(r)) for r in WRAP_RUNS] == [0, 0, 0, 0, -(1 << 62), MIN, 1 << 32, 1 << 32]


# ---- merge -----------------------------------------------------------------------
def merge_pair(rng, schema, na, nb):
    """Two batches; about 40 % of b's rows are rows of a whose weights cancel only mod 2^64 (2^63 + 2^63,
    2^62 + 3*2^62) or wrap to a non-zero total."""
    ca = [full_lane(rng, t, na, 0.5) for t in schema.lanes]
    wa = edge_weights(rng, na)
    a_cols, a_w = em.consolidate_np(schema, ca, wa)
    m = len(a_w)
    cb = [full_lane(rng, t, nb, 0.5) for t in schema.lanes]
    wb = edge_weights(rng, nb)
    if m:
        hit = rng.random(nb) < 0.4
        rows = rng.integers(0, m, int(hit.sum()))
        for c, ac in zip(cb, a_cols):
            c[hit] = ac[rows]
        aw = a_w[rows].view(np.uint64)
        cancel = rng.random(len(rows)) < 0.7   # partner weight = -w mod 2^64 (MIN + MIN, 2^62 + 3*2^62, ...)
        wb[hit] = np.where(cancel, (np.uint64(0) - aw), np.uint64(1) << np.uint64(63)).view(np.int64)
    b_cols, b_w = em.consolidate_np(schema, cb, wb)
    return (a_cols, a_w), (b_cols, b_w)


def run_merge_wrap(be, ref):
    rng = np.random.default_rng(47)
    for s in (Schema("u"), Schema("u", "u"), Schema("i", "i"), Schema("u", "uu"), Schema("i", "ui"),
              Schema("uiu", "uiuu")):
        for na, nb in ((1, 1), (3000, 2900), (100_000, 1000), (150_000, 170_000)):
            (ac, aw), (bc, bw) = merge_pair(rng, s, na, nb)
            exp = em.consolidate_np(s, [np.concatenate([x, y]) for x, y in zip(ac, bc)], np.concatenate([aw, bw]))
            check(be, ref, lambda b: b.merge(b.batch_from_sorted(s, ac, aw, len(aw), False),
                                             b.batch_from_sorted(s, bc, bw, len(bw), False)),
                  exp, f"merge {sid(s)} {na}+{nb}")


def run_merge_bounded(be, ref):
    rng = np.random.default_rng(53)
    cases = [(Schema("u", "i"), [MIN]), (Schema("u", "i"), [MAX]), (Schema("u", "i"), [-1]),
             (Schema("u", "u"), [UMAX]), (Schema("u", "u"), [1 << 63]), (Schema("i", "iu"), [MIN, UMAX]),
             (Schema("i", "iu"), [MAX, 0]), (Schema("u", "ui"), [UMAX, MIN])]
    for s, vb in cases:
        (ac, aw), (bc, bw) = merge_pair(rng, s, 60_000, 40_000)
        za = Z(s, zip(*[c.tolist() for c in ac], aw.tolist()))
        zb = Z(s, zip(*[c.tolist() for c in bc], bw.tolist()))
        exp = em.merge_bounded(za, zb, vb)
        mk = lambda b: (b.batch_from_sorted(s, ac, aw, len(aw), False), b.batch_from_sorted(s, bc, bw, len(bw), False))
        check(be, ref, lambda b: b.merge(*mk(b), val_lower_bound=vb), exp, f"merge_bounded {sid(s)} {vb}")

        def fuelled(b):
            m = b.merger(*mk(b), val_lower_bound=vb)
            while m.work(7919) <= 0:
                pass
            return m.done()

        check(be, ref, fuelled, exp, f"fuelled merger {sid(s)} {vb}")


def run_neg(be, ref):
    s = Schema("i", "u")
    rows = [(k, v, w) for k in I_POOL for v in U_POOL[:3] for w in W_POOL]
    z = Z(s, rows)
    check(be, ref, lambda b: b.neg(b.batch_from_rows(s, rows)), em.neg(z), "neg (-MIN = MIN)")


# ---- join and semijoin -----------------------------------------------------------
def join_inputs():
    ls, rs = Schema("i", "u"), Schema("i", "i")
    L = [(k, v, w) for k in I_POOL for v, w in zip(U_POOL, W_POOL[k % len(W_POOL):] + W_POOL)]
    R = [(k, v, w) for k in I_POOL for v, w in zip(I_POOL, W_POOL[::-1][(k * 3) % 5:] + W_POOL)]
    L += [(k, 5, 1 << 32) for k in (MIN, MAX)]
    R += [(k, 7, 1 << 32) for k in (MIN, MAX)]   # 2^32 * 2^32 = 0: the joined row must vanish
    return ls, rs, L, R


JOIN_PROJS = [
    Proj(Schema("i", "ui"), [key(0), lval(0), rval(0)]),
    Proj(Schema("i", "ui"), [key(0), lval(0), rval(0)], where=[lval(0).lt(rval(0))]),                # unsigned
    Proj(Schema("i", "ui"), [key(0), lval(0), rval(0)], where=[lval(0).lt(rval(0)).signed()]),       # signed
    Proj(Schema("ui", "i"), [lval(0), key(0), rval(0)], where=[rval(0).ge(0).signed(), key(0).gt(MAX - 1).signed()]),
    Proj(Schema("i", "u"), [key(0), lval(0) * rval(0)], where=[rval(0).le(1 << 63)]),
]


def run_join_batches(be, ref):
    ls, rs, L, R = join_inputs()
    zl, zr = Z(ls, L), Z(rs, R)
    for i, proj in enumerate(JOIN_PROJS):
        exp = em.join(zl, zr, proj)
        check(be, ref, lambda b: b.join_batches(b.batch_from_rows(ls, L), b.batch_from_rows(rs, R), proj), exp,
              f"join_batches proj {i}")
    zz = em.join(zl, zr, JOIN_PROJS[0])
    assert not any(r[0] in (MIN, MAX) and r[1] == 5 and r[2] == 7 for r in zz.rows())


def push_geometric(spines, bes, schema, n_batches, rows_of_batch, z=None):
    """Insert the same `n_batches` batches (geometrically shrinking, so that none merge) into one spine per backend;
    their rows are added to the model `z` when given."""
    for i in range(n_batches):
        cols, w = rows_of_batch(i)
        for sp, b in zip(spines, bes):
            sp.insert(b.batch_from_columns(schema, cols, w))
        if z is not None:
            z.add(zip(*[c.tolist() for c in cols], w.tolist()))


def deep_spine(bes, schema, n_batches, rows_of_batch):
    """New spines holding push_geometric's batches, and the model's union of them."""
    spines, z = [Spine(b, schema) for b in bes], Z(schema)
    push_geometric(spines, bes, schema, n_batches, rows_of_batch, z)
    return spines, z


def geometric_rows(schema, n_batches, seed):
    rng = np.random.default_rng(seed)

    def rows(i):
        n = 1 << (n_batches - 1 - i)
        j = np.arange(n, dtype=np.uint64)
        k = (j % np.uint64(61)) * np.uint64(0x0421_0842_1084_2108 + 2 * i + 1)   # spread over the full range
        cols = [k ^ em.SIGN if schema.key[0] == "i" else k]
        for l, t in enumerate(schema.lanes[1:]):
            v = (np.uint64(i) << np.uint64(56)) + j // np.uint64(61) + np.uint64(l)
            cols.append(v ^ em.SIGN if t == "i" else v)
        return cols, edge_weights(rng, n)

    return rows


def run_join_trace(be, ref):
    ts, ds = Schema("i", "ui"), Schema("i", "u")
    bes = [be] + ([ref] if ref is not None else [])
    rng = np.random.default_rng(59)
    for n_batches in (3, 18):
        spines, zt = deep_spine(bes, ts, n_batches, geometric_rows(ts, n_batches, 61 + n_batches))
        if n_batches > 16:
            assert spines[0].stats()[1] > 16, spines[0].stats()
        keys = sorted({t[0] for t in zt.d})
        D = [(keys[int(rng.integers(0, len(keys)))], em.u64(int(v)), int(w))
             for v, w in zip(full_lane(rng, "u", 400), edge_weights(rng, 400))]
        D += [(k, 1, 1 << 32) for k in keys[:3]] + [(MIN, 0, MIN), (MAX, UMAX, MAX)]
        zd = Z(ds, D)
        for left in (True, False):
            if left:
                proj = Proj(Schema("i", "uui"), [key(0), lval(0), rval(0), rval(1)], where=[rval(1).ge(0).signed()])
            else:
                proj = Proj(Schema("i", "uui"), [key(0), rval(0), lval(0), lval(1)], where=[rval(0).ge(1 << 63)])
            exp = em.join_delta_trace(zd, zt, proj, delta_is_left=left)
            got = be.join_delta_trace(be.batch_from_rows(ds, D), spines[0], proj, delta_is_left=left)
            em.assert_batch_is(got, exp, f"join_delta_trace {n_batches} batches left={left}")
            if ref is not None:
                other = ref.join_delta_trace(ref.batch_from_rows(ds, D), spines[1], proj, delta_is_left=left)
                assert_batches_equal(got, other, f"join_delta_trace {n_batches} batches left={left}: vs {ref.name}")


def run_semijoin(be, ref):
    ps, ks = Schema("i", "u"), Schema("i")
    P = [(k, v, w) for k in I_POOL for v, w in zip(U_POOL, W_POOL)]
    K = [(k, w) for k, w in zip(I_POOL, [1 << 32, MIN, -1, 1 << 62, 4, MAX, 1 << 32])]
    check(be, ref, lambda b: b.semijoin(b.batch_from_rows(ps, P), b.batch_from_rows(ks, K)),
          em.semijoin(Z(ps, P), Z(ks, K)), "semijoin")


# ---- the row language ------------------------------------------------------------
ARITH = Proj(Schema("i", "iiiiiii"), [key(0), -lval(0), lval(0) + lval(1), lval(0) - lval(1), lval(0) * lval(1),
                                      lval(0) // lval(1), lval(1) // lval(0), lval(0) // const(-1)])
U_AS_I = Proj(Schema("u", "iiu"), [key(0), lval(1) // lval(0), lval(1) // const(-1), lval(1) + const((1 << 63) + 5)])
CMPS = [capi.CMP_EQ, capi.CMP_NE, capi.CMP_LT, capi.CMP_LE, capi.CMP_GT, capi.CMP_GE]


def expr_rows():
    rows = [(i, a, b, 1) for i, (a, b) in enumerate((a, b) for a in I_POOL for b in I_POOL + [2, -2, 3, -3])]
    rows += [(1000 + i, a, b, 1) for i, (a, b) in enumerate([(7, 2), (-7, 2), (7, -2), (-7, -2), (MIN, 2), (MIN, -2)])]
    return rows


def run_map_index_arith(be, ref):
    s = Schema("i", "ii")
    rows = expr_rows()
    z = Z(s, rows)
    exp = em.map_index(z, ARITH)
    check(be, ref, lambda b: b.map_index(b.batch_from_rows(s, rows), ARITH), exp, "map_index arithmetic")
    # spot checks of the model itself: NEG MIN, MIN / -1, truncation toward zero, x / 0
    got = {r[0]: r[1:-1] for r in exp.rows()}
    for i, (a, b) in enumerate((a, b) for a in I_POOL for b in I_POOL + [2, -2, 3, -3]):
        if (a, b) == (MIN, -1):
            assert got[i][0] == MIN and got[i][4] == MIN and got[i][6] == MIN
        if b == 0:
            assert got[i][4] == 0
    assert [got[1000 + i][4] for i in range(6)] == [3, -3, -3, 3, MIN // 2, -(MIN // 2)]
    # u64 lanes >= 2^63 read as signed by DIV, constants >= 2^63
    s2 = Schema("u", "uu")
    rows2 = [(i, a, b, 1) for i, (a, b) in enumerate((a, b) for a in U_POOL + [2, 3] for b in U_POOL)]
    check(be, ref, lambda b: b.map_index(b.batch_from_rows(s2, rows2), U_AS_I), em.map_index(Z(s2, rows2), U_AS_I),
          "map_index u64 lanes as signed")


def run_predicates(be, ref):
    s = Schema("u", "u")
    vals = [0, 1, 63, 64, (1 << 63) - 2, (1 << 63) - 1, 1 << 63, (1 << 63) + 1, UMAX - 1, UMAX]
    rows = [(i, v, 1) for i, v in enumerate(vals)]
    z = Z(s, rows)
    out = Schema("u", "u")
    projs = []
    for c in CMPS:
        for bound in ((1 << 63) - 1, 1 << 63):
            for sg in (False, True):
                p = Pred(c, lval(0), const(bound), sg)
                projs.append((f"cmp {c} {bound} signed={sg}", Proj(out, [key(0), lval(0)], where=[p])))
    member = Pred(capi.CMP_IN, lval(0), const(em.w64((1 << 63) | (1 << 1) | 1)))   # codes {0, 1, 63}
    projs.append(("in {0,1,63}", Proj(out, [key(0), lval(0)], where=[member])))
    projs.append(("in, lval as code", Proj(out, [key(0), lval(0)], where=[Pred(capi.CMP_IN, lval(0), const(-1))])))
    for what, p in projs:
        exp = em.map_index(z, p)
        check(be, ref, lambda b: b.map_index(b.batch_from_rows(s, rows), p), exp, what)
    # CMP_IN is false for a >= 64 whatever the mask: a = 64 and 2^64-1 never pass
    assert [r[1] for r in em.map_index(z, projs[-1][1]).rows()] == [0, 1, 63]


def run_from_table(be, ref):
    rng = np.random.default_rng(67)
    n = 5000
    cols = [full_lane(rng, "i", n, 0.5), full_lane(rng, "u", n, 0.5), full_lane(rng, "i", n, 0.5)]
    w = edge_weights(rng, n)
    projs = [Proj(Schema("i", "iu"), [lval(0), lval(2) // lval(0), lval(1) * lval(2)]),
             Proj(Schema("u", "i"), [lval(1), -lval(0)], where=[lval(0).lt(lval(2)).signed(), lval(1).ge(1 << 63)]),
             Proj(Schema("i", "i"), [key(2), lval(0) - lval(2)], where=[lval(0).ne(MIN)])]
    for i, p in enumerate(projs):
        for wt in (None, w):
            exp = em.batch_from_table(cols, p, wt)
            check(be, ref, lambda b: b.batch_from_table(cols, p, wt), exp, f"batch_from_table proj {i} weights={wt is not None}")


# ---- weigh, aggregate_linear, average ---------------------------------------------
def run_weigh(be, ref):
    s = Schema("u", "i")
    rows = [(k, v, w) for k in (0, UMAX) for v in I_POOL for w in W_POOL[(v % 3):]]
    rows += [(7, 1 << 62, 4), (8, MIN, -1), (9, 3, 1 << 62), (9, 1, 1 << 62)]
    z = Z(s, rows)
    for mode in (capi.WEIGH_LINEAR, capi.WEIGH_AVG):
        for f in (lval(0), lval(0) * const(3), -key(0)):
            check(be, ref, lambda b: b.weigh(b.batch_from_rows(s, rows), f, mode), em.weigh(z, em_expr(f), mode),
                  f"weigh mode {mode}")


def em_expr(f):
    """`weigh` takes a Src or an Expr; the model evaluates Exprs."""
    from dbsp_b200.zset import _expr

    return _expr(f)


def avg_model(z):
    """apply_average of the integral: (k) -> sum / count, wrapping, truncating; no row where count == 0."""
    out = {}
    for k, vs in z.groups().items():
        s = em.w64(sum(v[0] * w for v, w in vs))
        c = em.w64(sum(w for _, w in vs))
        if c:
            q = em.expr(em_expr(const(s) // const(c)), ((), (), ()))
            out[k + (em.w64(q),)] = 1
    return out


def linear_model(z):
    out = {}
    for k, vs in z.groups().items():
        s = em.w64(sum(v[0] * w for v, w in vs))
        if s:
            out[k + (s,)] = 1
    return out


def zdiff(new, old):
    acc = dict(new)
    for t, w in old.items():
        acc[t] = acc.get(t, 0) - w
    return sorted(t + (w,) for t, w in acc.items() if w)


AVG_STEPS = [
    [(1, 5, 1), (1, 3, -1)],                                 # count 0, sum 2: no row
    [(2, 7, -2), (2, 1, -1)],                                # negative count: (-15) / (-3) = 5
    [(3, 7, 1), (3, 1, -3)],                                 # 4 / -2 = -2
    [(4, MIN, -1)],                                          # sum -MIN = MIN, count -1: MIN / -1 = MIN
    [(5, 1 << 62, 4), (5, 1, 1)],                            # sum wraps to 1, count 5: 0
    [(1, 0, 1), (6, 3, 1 << 62), (6, 3, 1 << 62), (6, 0, 1 << 62), (6, 0, 1 << 62)],   # key 6: count 0 by wrap
    [(2, 7, 2), (2, 1, 1), (4, 0, 1)],                       # key 2 gone; key 4 count 0 (sum MIN): its row leaves
    [(3, 1, 3), (4, 5, MAX)],
]


def run_average_and_linear(be, ref):
    s = Schema("u", "i")
    outs = {}
    for b in [be] + ([ref] if ref is not None else []):
        c = RootCircuit(b)
        a, h = c.add_input_indexed_zset(s)
        avg, lin = a.average(lval(0)).output(), a.aggregate_linear(lval(0)).output()
        got = []
        for rows in AVG_STEPS:
            h.append(rows)
            c.step()
            got.append((avg.value, lin.value))
        outs[b.name] = got
    z, pa, pl = Z(s), {}, {}
    for i, rows in enumerate(AVG_STEPS):
        z.add(rows)
        ca, cl = avg_model(z), linear_model(z)
        ga, gl = outs[be.name][i]
        assert [tuple(int(x) for x in r) for r in ga.rows()] == zdiff(ca, pa), ("average", i)
        assert [tuple(int(x) for x in r) for r in gl.rows()] == zdiff(cl, pl), ("aggregate_linear", i)
        if ref is not None:
            assert_batches_equal(ga, outs[ref.name][i][0], f"average step {i}: vs {ref.name}")
            assert_batches_equal(gl, outs[ref.name][i][1], f"aggregate_linear step {i}: vs {ref.name}")
        pa, pl = ca, cl
    assert avg_model(Z(s, AVG_STEPS[3]))[(4, MIN)] == 1 and avg_model(Z(s, AVG_STEPS[0])) == {}


# ---- aggregates --------------------------------------------------------------------
def agg_schemas(kind, in_schema):
    if kind in (capi.AGG_MAX, capi.AGG_MIN):
        return in_schema
    if kind == capi.AGG_WCOUNT:
        return Schema(in_schema.key, "i")
    return Schema(in_schema.key, "u")


def agg_steps(schema, kind, seed):
    """Batches of rows for the in-trace: extreme values, mixed-sign value tuples, and retractions in later batches
    that cancel the extreme candidates by +1/-1 and by wrap (2^63 + 2^63); key 0 loses more than 64 of them."""
    rng = np.random.default_rng(seed)
    nv = schema.nv
    ipool = I_POOL if schema.val[0] == "i" else U_POOL
    steps = []
    base = []
    for k in range(12):
        for j in range(10):
            v = [ipool[(k + j) % 7]] + [I_POOL[(j * 3 + l) % 7] if t == "i" else U_POOL[(j + l) % 7]
                                        for l, t in enumerate(schema.val[1:])]
            base.append((k,) + tuple(v) + (W_POOL[(k * 7 + j) % len(W_POOL)],))
    # key 0: 80 values at the top and the bottom of the range, weight 2^63 or 1
    ladder = [(0,) + (MAX - j if schema.val[0] == "i" else UMAX - j,) + (0,) * (nv - 1) + (MIN if j % 2 else 1,)
              for j in range(80)]
    ladder += [(0,) + (MIN + j if schema.val[0] == "i" else j,) + (0,) * (nv - 1) + (MIN if j % 2 else 1,)
               for j in range(80)]
    steps.append(base + ladder)
    # retract: 70 of the top and 70 of the bottom values of key 0, some extremes of other keys
    steps.append([r[:-1] + ((MIN if r[-1] == MIN else -1),) for r in ladder[:70] + ladder[80:150]]
                 + [r[:-1] + (em.w64(-r[-1]),) for r in base[::7]])
    steps.append([(k,) + tuple(int(full_lane(rng, t, 1)[0]) for t in schema.val) + (int(edge_weights(rng, 1)[0]),)
                  for k in range(12)])
    steps.append([r[:-1] + (em.w64(-r[-1]),) for r in base[3::5]])
    return steps


def run_aggregate(be, ref, kind, schema, deep):
    """The steps of agg_steps over a shallow trace (the Max / Min walk); `deep` then pushes 19 geometrically
    shrinking batches of other keys under the trace and retracts extremes one row per step, so that the trace stays
    above 16 batches (the general gather path) and some retractions cancel by wrap across batches."""
    bes = [be] + ([ref] if ref is not None else [])
    os_ = agg_schemas(kind, schema)
    ins = [Spine(b, schema) for b in bes]
    outs = [Spine(b, os_) for b in bes]
    zin, zout = Z(schema), Z(os_)
    depths = []

    def step(rows, i):
        delta = Z(schema, rows)
        zin.add(delta.rows())
        exp = em.aggregate_delta(delta, zin, zout, kind)
        res = []
        for sp, osp, b in zip(ins, outs, bes):
            d = b.batch_from_rows(schema, rows)
            sp.insert(d)
            res.append(b.aggregate_delta(d, sp, osp, kind))
            osp.insert(res[-1])
        depths.append(ins[0].stats()[1])
        what = f"aggregate kind {kind} {sid(schema)} step {i} over {depths[-1]} batches"
        em.assert_batch_is(res[0], exp, what)
        if ref is not None:
            assert_batches_equal(res[0], res[1], f"{what}: vs {ref.name}")
        zout.add(exp.rows())

    for i, rows in enumerate(agg_steps(schema, kind, 71 + kind)):
        step(rows, i)
    assert max(depths) <= 16
    if not deep:
        return
    def other_keys(i):   # keys 1000..: the model needs none of their rows, aggregate_delta reads the delta's keys only
        n = 1 << (18 - i)
        cols = [np.arange(1000, 1000 + n, dtype=np.uint64)] + [
            np.full(n, em.u64(I_POOL[i % 7] if t == "i" else U_POOL[i % 7]), np.uint64) for t in schema.val]
        return cols, np.full(n, 1 << 62, np.int64)

    push_geometric(ins, bes, schema, 19, other_keys)
    ipool = I_POOL if schema.val[0] == "i" else U_POOL
    tail = [(k % 6, ipool[k % 7]) + (0,) * (schema.nv - 1) + (MIN,) for k in range(10)]
    tail = tail + tail[::-1] + [(0, ipool[-1]) + (0,) * (schema.nv - 1) + (-1,)]
    for i, r in enumerate(tail):
        step([r], 100 + i)
    assert sum(d > 16 for d in depths[-len(tail):]) >= 3 * len(tail) // 4, depths


def run_wcount(be, ref):
    """aggregate_delta(WCOUNT) over an OrdZSet<K> with wrapping weights (the second half of aggregate_linear)."""
    bes = [be] + ([ref] if ref is not None else [])
    s, os_ = Schema("u"), Schema("u", "i")
    ins, outs = [Spine(b, s) for b in bes], [Spine(b, os_) for b in bes]
    zin, zout = Z(s), Z(os_)
    steps = [[(k, W_POOL[k % len(W_POOL)]) for k in range(20)] + [(UMAX, MAX)],
             [(k, W_POOL[(k + 3) % len(W_POOL)]) for k in range(20)] + [(UMAX, 1)],
             [(k, MIN) for k in range(0, 20, 2)] + [(UMAX, MAX)]]
    for i, rows in enumerate(steps):
        delta = Z(s, rows)
        zin.add(delta.rows())
        exp = em.aggregate_delta(delta, zin, zout, capi.AGG_WCOUNT)
        res = []
        for sp, osp, b in zip(ins, outs, bes):
            d = b.batch_from_rows(s, rows)
            sp.insert(d)
            res.append(b.aggregate_delta(d, sp, osp, capi.AGG_WCOUNT))
            osp.insert(res[-1])
        em.assert_batch_is(res[0], exp, f"wcount step {i}")
        if ref is not None:
            assert_batches_equal(res[0], res[1], f"wcount step {i}: vs {ref.name}")
        zout.add(exp.rows())


# ---- distinct ----------------------------------------------------------------------
def run_distinct(be, ref):
    s = Schema("i", "u")
    integral_rows = [(k, v, w) for k in (MIN, -1, 0, MAX) for v, w in zip((0, 1, UMAX, 1 << 63, 5, 6),
                                                                          (MAX, MIN, MAX - 1, MIN + 1, 1, -1))]
    zi = Z(s, integral_rows)
    deltas = [(k, v, d) for k in (MIN, -1, 0, MAX) for v, d in zip((0, 1, UMAX, 1 << 63, 5, 6, 9),
                                                                   (1, -1, 1, -1, MAX, MIN, MIN))]
    zd = Z(s, deltas)
    exp = em.distinct_delta(zd, zi)
    assert exp.d[(MIN, 0)] == -1 and exp.d[(MIN, 1)] == 1   # MAX + 1 wraps to MIN; MIN - 1 wraps to MAX

    def op(b):
        sp = Spine(b, s)
        sp.insert(b.batch_from_rows(s, integral_rows))
        return b.distinct_delta(b.batch_from_rows(s, deltas), sp)

    check(be, ref, op, exp, "distinct_delta across the sign by wrap")
    check(be, ref, lambda b: b.stream_distinct(b.batch_from_rows(s, integral_rows + deltas)),
          em.stream_distinct(em.union(zi, zd)), "stream_distinct")


# ---- bounds ------------------------------------------------------------------------
def bound_rows(t):
    pool = I_POOL if t == "i" else U_POOL
    return [(k, v, W_POOL[(i + j) % len(W_POOL)]) for i, k in enumerate(pool) for j, v in enumerate((0, 1, UMAX))]


def run_bounds(be, ref):
    for t in "iu":
        s = Schema(t, "u")
        rows = bound_rows(t)
        z = Z(s, rows)
        pool = I_POOL if t == "i" else U_POOL
        for bnd in pool:
            exp = em.truncate_keys_below(z, [bnd])
            check(be, ref, lambda b: b.truncate_keys_below(b.batch_from_rows(s, rows), [bnd]), exp,
                  f"batch truncate_keys_below {t} {bnd}")

            def spine_trunc(b):
                sp = Spine(b, s)
                sp.insert(b.batch_from_rows(s, rows[::2]))
                sp.truncate_keys_below([bnd])
                sp.insert(b.batch_from_rows(s, rows[1::2]))   # later inserts are truncated too
                return sp.consolidate()

            check(be, ref, spine_trunc, exp, f"spine truncate_keys_below {t} {bnd}")
        for vb in (0, 1 << 63, UMAX):
            exp = em.merge_bounded(z, Z(s), [vb])

            def spine_vals(b):
                sp = Spine(b, s)
                sp.insert(b.batch_from_rows(s, rows))
                sp.truncate_values_below([vb])
                return sp.consolidate()

            check(be, ref, spine_vals, exp, f"truncate_values_below {t} {vb}")
        for bs in (be, ref):
            if bs is not None:
                assert bs.batch_from_rows(s, rows).last_key() == em.last_key(z)
                assert bs.batch_from_rows(s, [r for r in rows if r[0] != pool[-1]]).last_key() == (pool[-2],)
        # windows with bounds at the extremes
        # bounds only grow, except that the end may move back (window.rs); the last window is empty
        wins = [None, (pool[0], pool[1]), (pool[0], pool[3]), (pool[2], pool[-1]), (pool[3], pool[-2]),
                (pool[-1], pool[-1])]
        delta_rows = [(k, 2, 1) for k in pool] + [(pool[0], 3, MIN)]
        zd = Z(s, delta_rows)
        for prev, cur in zip(wins, wins[1:]):
            exp = em.window_delta(z, zd, None if prev is None else ([prev[0]], [prev[1]]), ([cur[0]], [cur[1]]))

            def win(b):
                sp = Spine(b, s)
                sp.insert(b.batch_from_rows(s, rows))
                return b.window_delta(sp, b.batch_from_rows(s, delta_rows),
                                      None if prev is None else ([prev[0]], [prev[1]]), ([cur[0]], [cur[1]]))

            check(be, ref, win, exp, f"window {t} {prev} -> {cur}")


def run_shards(be, ref):
    for s in (Schema("i", "u"), Schema("u", "i"), Schema("iu")):
        rng = np.random.default_rng(73)
        n = 20_000
        cols = [full_lane(rng, t, n, 0.5) for t in s.lanes]
        w = edge_weights(rng, n)
        exp = em.consolidate_np(s, cols, w)
        b = be.batch_from_columns(s, cols, w)
        for n_shards in (1, 3, 8):
            parts = be.shard_partition(b, n_shards)
            acc = be.batch_empty(s)
            for p in parts:
                acc = be.merge(acc, p)
            em.assert_batch_is(acc, exp, f"union of {n_shards} shards {sid(s)}")
            if ref is not None:
                rparts = ref.shard_partition(ref.batch_from_columns(s, cols, w), n_shards)
                for i, (p, q) in enumerate(zip(parts, rparts)):
                    assert_batches_equal(p, q, f"shard {i} of {n_shards}: vs {ref.name}")


ALL_CASES = {}
for _s in SCHEMAS:
    for _n in (1, 31, 3073, 6145, 70_001):
        ALL_CASES[f"consolidate_full_{sid(_s)}_{_n}"] = lambda be, ref=None, s=_s, n=_n: run_consolidate_full(be, ref, s, n, n + 7)
for _s in (Schema("u", "u"), Schema("i", "u"), Schema("uiu", "uiuu")):
    for _n in (300_000, 1_000_003):
        ALL_CASES[f"consolidate_full_{sid(_s)}_{_n}"] = lambda be, ref=None, s=_s, n=_n: run_consolidate_full(be, ref, s, n, n + 7)
ALL_CASES.update({
    "consolidate_plans": lambda be, ref=None: run_consolidate_plans(be, ref),
    "wrap_runs": lambda be, ref=None: run_wrap_runs(be, ref),
    "merge_wrap": lambda be, ref=None: run_merge_wrap(be, ref),
    "merge_bounded": lambda be, ref=None: run_merge_bounded(be, ref),
    "neg": lambda be, ref=None: run_neg(be, ref),
    "join_batches": lambda be, ref=None: run_join_batches(be, ref),
    "join_trace": lambda be, ref=None: run_join_trace(be, ref),
    "semijoin": lambda be, ref=None: run_semijoin(be, ref),
    "map_index_arith": lambda be, ref=None: run_map_index_arith(be, ref),
    "predicates": lambda be, ref=None: run_predicates(be, ref),
    "from_table": lambda be, ref=None: run_from_table(be, ref),
    "weigh": lambda be, ref=None: run_weigh(be, ref),
    "average_and_linear": lambda be, ref=None: run_average_and_linear(be, ref),
    "wcount": lambda be, ref=None: run_wcount(be, ref),
    "distinct": lambda be, ref=None: run_distinct(be, ref),
    "bounds": lambda be, ref=None: run_bounds(be, ref),
    "shards": lambda be, ref=None: run_shards(be, ref),
})
AGG_NAMES = {capi.AGG_MAX: "max", capi.AGG_MIN: "min", capi.AGG_FOLD_COUNT: "count", capi.AGG_FOLD_SUM: "sum"}
_AGG = [(k, s, False) for k in AGG_NAMES for s in (Schema("u", "i"), Schema("u", "iu"), Schema("u", "u"))]
_AGG += [(capi.AGG_MAX, Schema("u", "i"), True), (capi.AGG_MIN, Schema("u", "iu"), True),
         (capi.AGG_FOLD_SUM, Schema("u", "u"), True)]
for _k, _s, _deep in _AGG:
    ALL_CASES[f"aggregate_{AGG_NAMES[_k]}_{sid(_s)}_{'deep' if _deep else 'shallow'}"] = (
        lambda be, ref=None, k=_k, s=_s, d=_deep: run_aggregate(be, ref, k, s, d))
