"""Backend-generic tests of the ABI's error contract (include/dbsp_b200.h, DESIGN §1): an argument or a snapshot file
a host can get wrong is refused on the host, before anything is allocated, copied or launched.

Every case has three parts, and all three are asserted:
  1. the refusal: the status, and a dbsp_last_error text naming the call and the argument;
  2. nothing ran: the context's launch, copy and host-wait counters are unchanged and the out-pointer is still NULL;
  3. the nearest accepted input: the same call with the offending value moved to the last legal one, compared with
     the exact model (tests/exact_model.py) and, given a second backend, bit for bit with it.  This keeps the
     validators from being too strict and puts the kernels at their argument limits.
The calls go through `CApi` directly wherever the Python wrappers of zset.py would stop the bad value first.
After every group one valid operator call on the same context is compared with the model: a refusal leaves the
context usable and the error text does not stick to the calls that follow."""
import ctypes as C
import os
import struct

import numpy as np

import exact_model as em
import snapshot_cases
from dbsp_b200 import Proj, Schema, Spine, capi, const, key, lval, rval
from dbsp_b200._capi import CExpr, CProj, CSchema, as_u64, col_ptrs
from dbsp_b200.zset import Expr, Pred, Src, _expr, _lanes
from edge_cases import SCHEMAS, check, sid
from exact_model import Z
from parity_util import assert_batches_equal
from trace_cases import rand_rows, signed_rows

INVALID, UNSUPPORTED = 1, 4


# ---- the harness -------------------------------------------------------------------------------------------------
def counters(be):
    s = be.stats()
    return s["kernel_launches"], s["h2d_bytes"], s["d2h_bytes"], s["host_waits"]


def refused(be, call, *args, names, status=INVALID, outs=(), ran_nothing=True, call_named=True):
    """The raw call returns `status`, names itself and `names` in the error text, touched no out-pointer and (unless
    the case says the file had to be read first) neither launched, copied nor waited."""
    before = counters(be)
    rc = getattr(be.api, "_" + call)(*args)
    msg = (be.api._last_error() or b"").decode()
    assert rc == status, f"{call}: status {rc}, expected {status} ({msg!r})"
    assert call in msg or not call_named, f"{call}: the error text does not name the call: {msg!r}"
    for n in ([names] if isinstance(names, str) else names):
        assert n in msg, f"{call}: the error text does not name {n!r}: {msg!r}"
    for o in outs:
        assert not o.value, f"{call}: a refused call wrote its out-pointer"
    if ran_nothing:
        assert counters(be) == before, f"{call}: a refused call launched, copied or waited: {before} -> {counters(be)}"
    return msg


def out():
    return C.c_void_p()


def cschema(nk, nv, types=()):
    s = CSchema()
    s.n_key_lanes, s.n_val_lanes = nk, nv
    for i, t in enumerate(types):
        s.lane_types[i] = t
    return s


def mutated(proj, fn):
    """A copy of the C struct of `proj` with fn applied: values the Proj class would not build."""
    c = CProj.from_buffer_copy(proj._c)
    fn(c)
    return C.byref(c)


def rows_of(rng, s, n, hi=40):
    return rand_rows(rng, n, hi, hi, 3, nk=s.nk, nv=s.nv)


def still_usable(be, ref, what):
    """One valid operator call after a group of refusals, against the model."""
    s = Schema("u", "u")
    rows = [(1, 2, 3), (1, 2, -1), (4, 5, 1), (0, 9, 2)]
    p = Proj(Schema("u", "u"), [lval(0), key(0) + 1], where=[key(0).lt(4)])
    check(be, ref, lambda b: b.map_index(b.batch_from_rows(s, rows), p), em.map_index(Z(s, rows), p), f"usable after {what}")


# ---- schema ------------------------------------------------------------------------------------------------------
BAD_SCHEMAS = {
    "no lanes": (cschema(0, 0), "1..8 lanes"),
    "nine lanes": (cschema(5, 4), "1..8 lanes"),
    "lane count wrapping uint8": (cschema(200, 57), "1..8 lanes"),   # 257: one lane if summed in a uint8
    "lane type 2": (cschema(1, 1, (0, 2)), "lane_types[1]"),
}


def run_schema(be, ref=None):
    one = np.array([7], dtype=np.uint64)
    cols, w = col_ptrs([one] * 8), np.array([1], dtype=np.int64)
    base = be.batch_from_rows(Schema("u", "u"), [(1, 2, 1)])
    for what, (cs, names) in BAD_SCHEMAS.items():
        o = out()
        refused(be, "batch_from_tuples", be.ctx, C.byref(cs), cols, w.ctypes.data, 1, 0, C.byref(o), names=["schema", names], outs=[o])
        refused(be, "batch_from_sorted", be.ctx, C.byref(cs), cols, w.ctypes.data, 1, 0, C.byref(o), names=["schema", names], outs=[o])
        refused(be, "batch_empty", be.ctx, C.byref(cs), C.byref(o), names=["schema", names], outs=[o])
        refused(be, "batcher_new", be.ctx, C.byref(cs), C.byref(o), names=["schema", names], outs=[o])
        refused(be, "spine_new", be.ctx, C.byref(cs), C.byref(o), names=["schema", names], outs=[o])
        p = Proj(Schema("u", "u"), [key(0), lval(0)])
        bad = mutated(p, lambda c: setattr(c, "out_schema", cs))
        refused(be, "map_index", be.ctx, base.h, bad, C.byref(o), names=["proj.out_schema", names], outs=[o])
    # accepted: 1 and 8 lanes, in every constructor
    rng = np.random.default_rng(3)
    for s in (Schema("i"), Schema("u"), Schema("uiu", "iuiui"), Schema("uuuuuuuu"), Schema("u", "iiiiiii")):
        rows = rows_of(rng, s, 300)
        z = Z(s, rows)
        check(be, ref, lambda b: b.batch_from_rows(s, rows), z, f"from_tuples {sid(s)}")
        fc, fw = em.flat(s, z)
        check(be, ref, lambda b: b.batch_from_sorted(s, fc, fw, len(fw), False), z, f"from_sorted {sid(s)}")
        assert len(be.batch_empty(s)) == 0 and be.batch_empty(s).schema == s

        def through_batcher(b):
            q = b.batcher(s)
            q.push_rows(rows[:100])
            q.push_rows(rows[100:])
            return q.seal()

        def through_spine(b):
            tr = Spine(b, s)
            tr.insert(b.batch_from_rows(s, rows[:100]))
            tr.insert(b.batch_from_rows(s, rows[100:]))
            return tr.consolidate()

        check(be, ref, through_batcher, z, f"batcher {sid(s)}")
        check(be, ref, through_spine, z, f"spine {sid(s)}")
    still_usable(be, ref, "schema refusals")


# ---- projections and expressions -----------------------------------------------------------------------------------
ALL_OPS = [capi.OP_COPY, capi.OP_NEG, capi.OP_ADD, capi.OP_SUB, capi.OP_MUL, capi.OP_DIV]


def run_proj(be, ref=None):
    rng = np.random.default_rng(5)
    s = Schema("ui", "uiu")   # 2 key lanes, 3 value lanes
    rows = rows_of(rng, s, 400)
    z = Z(s, rows)
    b = be.batch_from_rows(s, rows)
    rb = ref.batch_from_rows(s, rows) if ref is not None else None
    pick = lambda x: b if x is be else rb
    os2 = Schema("u", "u")
    o = out()

    # map_index: one past the last lane of each source; SRC_RVAL reads the value lanes like SRC_LVAL (one input)
    for src, names in ((key(2), "SRC_KEY has 2"), (lval(3), "SRC_LVAL has 3"), (rval(3), "SRC_RVAL has 3"), (key(255), "SRC_KEY")):
        for p in (Proj(os2, [src, const(0)]), Proj(os2, [const(0), const(1) + src]), Proj(os2, [const(0), const(0)], where=[src.eq(1)]),
                  Proj(os2, [const(0), const(0)], where=[const(1).eq(src)])):
            refused(be, "map_index", be.ctx, b.h, p.c(), C.byref(o), names=["idx", names], outs=[o])
    good = Proj(os2, [key(0), lval(0)], where=[key(1).ge(0).signed()])
    for what, fn, names in (
        ("kind 4", lambda c: setattr(c.out[0].a, "kind", 4), "proj.out[0].a.kind"),
        ("kind 4 in a predicate", lambda c: setattr(c.pred[0].b, "kind", 4), "proj.pred[0].b.kind"),
        ("op 6", lambda c: setattr(c.out[1], "op", 6), "proj.out[1].op"),
        ("cmp 7", lambda c: setattr(c.pred[0], "cmp", 7), "proj.pred[0].cmp"),
        ("n_pred 5", lambda c: setattr(c, "n_pred", 5), "proj.n_pred"),
        ("n_pred 255", lambda c: setattr(c, "n_pred", 255), "proj.n_pred"),
    ):
        refused(be, "map_index", be.ctx, b.h, mutated(good, fn), C.byref(o), names=names, outs=[o])
    # accepted: the last lane of each source, 8 output lanes, 4 predicates
    last = Proj(Schema("uiu", "uiuiu"), [key(1), lval(2), rval(2), key(0), lval(0), rval(1), const(-1), key(1) - lval(1)],
                where=[key(1).ge(-30).signed(), lval(2).lt(35), rval(2).ne(7), key(0).isin([1, 2, 3, 5, 8, 13, 21, 34])])
    check(be, ref, lambda x: x.map_index(pick(x), last), em.map_index(z, last), "map_index at the last lanes, 8 out lanes, 4 predicates")
    # every operation over every pair of source kinds
    srcs = [key(1), lval(2), rval(1), const(-3)]
    for op in ALL_OPS:
        for a in srcs:
            outs8 = [Expr(op, a, bb) for bb in srcs] + [Expr(op, bb, a) for bb in srcs]
            p = Proj(Schema("iiii", "iiii"), outs8)
            check(be, ref, lambda x: x.map_index(pick(x), p), em.map_index(z, p), f"op {op} over every source kind")
    # CMP_IN at its edges: a = 63 is the last member a mask can hold, a = 64 never matches
    sin = Schema("u", "i")
    in_rows = [(a, m, 1) for a in (0, 1, 62, 63, 64, 65, 1 << 32, em.UMAX) for m in (-1, em.MIN, em.MAX, 1, 0)]
    pin = Proj(sin, [key(0), lval(0)], where=[Pred(capi.CMP_IN, key(0), lval(0))])
    zin = Z(sin, in_rows)
    got = check(be, ref, lambda x: x.map_index(x.batch_from_rows(sin, in_rows), pin), em.map_index(zin, pin), "CMP_IN at a = 63 / 64")
    assert (63, em.MIN, 1) in got.rows() and (63, -1, 1) in got.rows() and not any(r[0] >= 64 for r in got.rows())

    # raw tables: every source kind names a column
    ncols, n = 3, 500
    tcols = [rng.integers(0, 50, n).astype(np.uint64) for _ in range(ncols)]
    tw = rng.integers(-2, 3, n).astype(np.int64)
    ptrs = col_ptrs(tcols)
    for mk in (key, lval, rval):
        bad = Proj(os2, [mk(0), mk(3)])
        refused(be, "batch_from_table", be.ctx, ptrs, ncols, tw.ctypes.data, n, 0, bad.c(), C.byref(o), names=["idx", "has 3"], outs=[o])
    tlast = Proj(Schema("u", "uu"), [key(2), lval(2) + rval(2), rval(0)], where=[lval(2).ge(5)])
    check(be, ref, lambda x: x.batch_from_table(tcols, tlast, tw), em.batch_from_table(tcols, tlast, tw), "from_table at the last column")
    # a masked upload: the projection may read exactly the uploaded columns
    up = be.upload_begin(tcols, 0b101, tw)
    refused(be, "batch_from_upload", be.ctx, up.h, Proj(os2, [lval(0), lval(1)]).c(), C.byref(o), names=["column 1", "col_mask"], outs=[o])
    refused(be, "batch_from_upload", be.ctx, up.h, Proj(os2, [lval(0), lval(3)]).c(), C.byref(o), names=["idx", "has 3"], outs=[o])
    masked = Proj(Schema("u", "u"), [lval(2), key(0) * 3], where=[rval(0).ne(rval(2))])
    assert be.proj_table_mask(masked) == 0b101
    expect = em.batch_from_table(tcols, masked, tw)
    em.assert_batch_is(be.batch_from_upload(up, masked), expect, "from_upload reading exactly the unmasked columns")
    if ref is not None:
        assert_batches_equal(be.batch_from_upload(be.upload_begin(tcols, 0b101, tw), masked),
                             ref.batch_from_upload(ref.upload_begin(tcols, 0b101, tw), masked), "from_upload vs the second backend")

    # joins: the key, the left values and the right values have their own lane counts
    ls, rs = Schema("i", "uu"), Schema("i", "u")
    lrows, rrows = rows_of(rng, ls, 300, 25), rows_of(rng, rs, 300, 25)
    zl, zr = Z(ls, lrows), Z(rs, rrows)
    js = Schema("i", "uu")

    def join_inputs(x):
        tl, tr = Spine(x, ls), Spine(x, rs)
        tl.insert(x.batch_from_rows(ls, lrows))
        tr.insert(x.batch_from_rows(rs, rrows))
        return x.batch_from_rows(ls, lrows), x.batch_from_rows(rs, rrows), tl, tr

    bl, br, tl, tr = join_inputs(be)
    for src, names in ((key(1), "SRC_KEY has 1"), (lval(2), "SRC_LVAL has 2"), (rval(1), "SRC_RVAL has 1")):
        bad = Proj(js, [key(0), src, const(0)])
        refused(be, "join_batches", be.ctx, bl.h, br.h, bad.c(), C.byref(o), names=["idx", names], outs=[o])
        refused(be, "join_delta_trace", be.ctx, bl.h, tr.h, bad.c(), 1, C.byref(o), names=["idx", names], outs=[o])
        refused(be, "join_delta_trace", be.ctx, br.h, tl.h, bad.c(), 0, C.byref(o), names=["idx", names], outs=[o])   # delta feeds SRC_RVAL
    refused(be, "join_batches", be.ctx, bl.h, br.h, None, C.byref(o), names="proj is NULL", outs=[o])
    jlast = Proj(js, [key(0), lval(1), rval(0)], where=[lval(0).le(rval(0))])
    ej = em.join(zl, zr, jlast)
    check(be, ref, lambda x: (lambda i: x.join_batches(i[0], i[1], jlast))(join_inputs(x)), ej, "join_batches at the last lanes")
    check(be, ref, lambda x: (lambda i: x.join_delta_trace(i[0], i[3], jlast, True))(join_inputs(x)), ej, "join_delta_trace, delta left")
    check(be, ref, lambda x: (lambda i: x.join_delta_trace(i[1], i[2], jlast, False))(join_inputs(x)), ej, "join_delta_trace, delta right")

    # weigh: f reads the key and the values of the one input
    for src, names in ((key(2), "SRC_KEY has 2"), (lval(3), "SRC_LVAL has 3"), (rval(3), "SRC_RVAL has 3")):
        refused(be, "weigh", be.ctx, b.h, C.byref(_expr(src).c()), capi.WEIGH_LINEAR, C.byref(o), names=["f", "idx", names], outs=[o])
    e6 = CExpr()
    e6.op = 6
    refused(be, "weigh", be.ctx, b.h, C.byref(e6), capi.WEIGH_LINEAR, C.byref(o), names="f.op", outs=[o])
    refused(be, "weigh", be.ctx, b.h, None, capi.WEIGH_LINEAR, C.byref(o), names="f is NULL", outs=[o])
    for f in (lval(2) * key(1), rval(2) - 1):
        for mode in (capi.WEIGH_LINEAR, capi.WEIGH_AVG):
            check(be, ref, lambda x: x.weigh(pick(x), f, mode), em.weigh(z, _expr(f), mode), f"weigh at the last lanes, mode {mode}")
    still_usable(be, ref, "projection refusals")


# ---- operand pairs ---------------------------------------------------------------------------------------------------
def run_pairs(be, ref=None):
    rng = np.random.default_rng(7)
    o = out()
    keep = []   # a handle passed as `x.h` must outlive the call: the wrappers free theirs when collected

    def mk(s, n=60):
        keep.append(be.batch_from_rows(s, rows_of(rng, s, n, 12)))
        return keep[-1]

    def spine_of(s, n=60, fill=True):
        t = Spine(be, s)
        keep.append(t)
        if fill:
            t.insert(mk(s, n))
        return t

    u_u, uu_u, i_u, u, uu, u_uu = Schema("u", "u"), Schema("uu", "u"), Schema("i", "u"), Schema("u"), Schema("uu"), Schema("u", "uu")
    pj = Proj(Schema("u"), [key(0)])
    kl = "key lanes"
    for other in (uu_u, i_u):   # a key lane more; the same count with another type
        refused(be, "join_batches", be.ctx, mk(u_u).h, mk(other).h, pj.c(), C.byref(o), names=kl, outs=[o])
        refused(be, "join_delta_trace", be.ctx, mk(u_u).h, spine_of(other).h, pj.c(), 1, C.byref(o), names=kl, outs=[o])
        refused(be, "join_delta_trace", be.ctx, mk(other).h, spine_of(u_u).h, pj.c(), 0, C.byref(o), names=kl, outs=[o])
        refused(be, "semijoin", be.ctx, mk(u_u).h, mk(Schema(other.key)).h, C.byref(o), names=["keys", kl], outs=[o])
        refused(be, "distinct_delta", be.ctx, mk(u_u).h, spine_of(other).h, C.byref(o), names=["delayed_integral", "schema"], outs=[o])
        b4 = _lanes([0]), _lanes([5]), _lanes([1]), _lanes([7])
        refused(be, "window_delta", be.ctx, spine_of(other).h, mk(u_u).h, 1, *b4, C.byref(o), names=["trace", "schema"], outs=[o])
        refused(be, "batch_merge", be.ctx, mk(u_u).h, mk(other).h, C.byref(o), names=["a and b", "schema"], outs=[o])
        refused(be, "batch_merge_bounded", be.ctx, mk(u_u).h, mk(other).h, None, C.byref(o), names=["a and b", "schema"], outs=[o])
        refused(be, "merger_new", be.ctx, mk(u_u).h, mk(other).h, None, C.byref(o), names=["a and b", "schema"], outs=[o])
        refused(be, "spine_insert", be.ctx, spine_of(u_u).h, mk(other).h, names=["batch", "schema"])
    refused(be, "semijoin", be.ctx, mk(u_u).h, mk(u_u).h, C.byref(o), names=["keys", "value lanes"], outs=[o])
    refused(be, "distinct_delta", be.ctx, mk(u_u).h, spine_of(u_uu).h, C.byref(o), names="schema", outs=[o])   # the integral's rows are wider

    # aggregate_delta: delta / in_trace / out_trace must fit each other and the aggregator
    A = capi
    agg = lambda d, i, t, kind, names: refused(be, "aggregate_delta", be.ctx, mk(d).h, spine_of(i).h, spine_of(t, fill=False).h, kind, C.byref(o),
                                               names=names, outs=[o])
    agg(u_u, u_u, u_u, -1, "agg_kind")
    agg(u_u, u_u, u_u, 6, "agg_kind")
    agg(u_u, uu_u, u_u, A.AGG_MAX, ["delta", "in_trace"])
    agg(u_u, u_uu, u_u, A.AGG_MAX, ["delta", "in_trace"])
    agg(u_u, u_u, uu_u, A.AGG_MAX, ["out_trace", "key lanes"])
    agg(u_u, u_u, i_u, A.AGG_MIN, ["out_trace", "key lanes"])
    agg(u_u, u_u, u_uu, A.AGG_MAX, ["AGG_MAX", "out_trace"])          # the output has a value lane more than the input
    agg(u_u, u_u, Schema("u", "i"), A.AGG_MIN, "value lane types")
    agg(u, u, u_u, A.AGG_MAX, "AGG_MAX")                               # nothing to take the maximum of
    agg(u, u, u_u, A.AGG_FOLD_COUNT, "AGG_FOLD")                       # FOLD_* fold the values
    agg(u, u, u_u, A.AGG_FOLD_SUM, "AGG_FOLD")
    agg(u_u, u_u, u_uu, A.AGG_FOLD_SUM, "one value lane")
    agg(u_u, u_u, Schema("u", "i"), A.AGG_WCOUNT, "AGG_WCOUNT")        # WCOUNT counts the weights of an OrdZSet<K>
    agg(u_u, u_u, u_uu, A.AGG_WCOUNT2, "AGG_WCOUNT2")
    agg(uu, uu, u_u, A.AGG_WCOUNT2, "AGG_WCOUNT2")                     # (sum, count) are two lanes
    agg(uu, uu, Schema("uu", "ii"), A.AGG_WCOUNT2, "AGG_WCOUNT2")      # the key is (K.., which) minus `which`
    refused(be, "weigh", be.ctx, mk(u_u).h, C.byref(_expr(lval(0)).c()), 2, C.byref(o), names="mode", outs=[o])
    refused(be, "weigh", be.ctx, mk(u_u).h, C.byref(_expr(lval(0)).c()), -1, C.byref(o), names="mode", outs=[o])
    refused(be, "weigh", be.ctx, mk(Schema("uuuuuuuu")).h, C.byref(_expr(key(0)).c()), capi.WEIGH_AVG, C.byref(o), names="WEIGH_AVG", outs=[o])
    # a bound that is required
    refused(be, "batch_truncate_keys_below", be.ctx, mk(u_u).h, None, C.byref(o), names="key is NULL", outs=[o])
    refused(be, "spine_truncate_keys_below", be.ctx, spine_of(u_u).h, None, names="key is NULL")
    refused(be, "spine_truncate_values_below", be.ctx, spine_of(u_u).h, None, names="val is NULL")
    refused(be, "window_delta", be.ctx, spine_of(u_u).h, mk(u_u).h, 1, None, None, _lanes([1]), _lanes([7]), C.byref(o), names="start0", outs=[o])
    refused(be, "window_delta", be.ctx, spine_of(u_u).h, mk(u_u).h, 0, None, None, None, _lanes([7]), C.byref(o), names="start1", outs=[o])

    # accepted: every operator of the group on operands that fit, at the edge of what fits
    s = Schema("ui", "u")
    ra, rb_ = rows_of(rng, s, 200, 12), rows_of(rng, s, 200, 12)
    za, zb = Z(s, ra), Z(s, rb_)
    rk = rows_of(rng, Schema("ui"), 60, 12)
    pair = lambda x: (x.batch_from_rows(s, ra), x.batch_from_rows(s, rb_))

    def tr_of(x, rows, sch=s):
        t = Spine(x, sch)
        t.insert(x.batch_from_rows(sch, rows))
        return t

    check(be, ref, lambda x: x.semijoin(x.batch_from_rows(s, ra), x.batch_from_rows(Schema("ui"), rk)), em.semijoin(za, Z(Schema("ui"), rk)), "semijoin")
    check(be, ref, lambda x: x.distinct_delta(x.batch_from_rows(s, ra), tr_of(x, rb_)), em.distinct_delta(za, zb), "distinct_delta")
    prev, cur = ([2, -5], [9, 3]), ([4, 0], [11, 0])
    check(be, ref, lambda x: x.window_delta(tr_of(x, rb_), x.batch_from_rows(s, ra), prev, cur), em.window_delta(zb, za, prev, cur), "window_delta")
    check(be, ref, lambda x: x.window_delta(tr_of(x, rb_), x.batch_from_rows(s, ra), None, cur), em.window_delta(zb, za, None, cur),
          "window_delta without a previous window (start0 / end0 not needed)")
    check(be, ref, lambda x: x.merge(*pair(x)), em.union(za, zb), "merge")
    check(be, ref, lambda x: x.merge(*pair(x), val_lower_bound=[6]), em.merge_bounded(za, zb, [6]), "merge_bounded")
    o2, (pa, pb) = out(), pair(be)
    be.api.call("batch_merge_bounded", be.ctx, pa.h, pb.h, None, C.byref(o2))   # NULL = no bound
    from dbsp_b200.zset import Batch
    em.assert_batch_is(Batch(be, o2.value, s), em.union(za, zb), "merge_bounded without a bound")
    zin = em.union(za, zb)
    for kind, osch in ((A.AGG_MAX, s), (A.AGG_MIN, s), (A.AGG_FOLD_COUNT, Schema("ui", "u")), (A.AGG_FOLD_SUM, Schema("ui", "u"))):
        def run(x, kind=kind, osch=osch):
            tin = tr_of(x, rb_)
            d = x.batch_from_rows(s, ra)
            tin.insert(d)
            return x.aggregate_delta(d, tin, Spine(x, osch), kind)
        check(be, ref, run, em.aggregate_delta(za, zin, Z(osch), kind), f"aggregate kind {kind}")
    # WCOUNT over keys only, WCOUNT2 over (K.., which) rows
    ks, ko = Schema("ui"), Schema("ui", "i")
    wa = em.weigh(za, _expr(lval(0)), capi.WEIGH_LINEAR)
    check(be, ref, lambda x: (lambda d: x.aggregate_delta(d, tr_of(x, wa.rows(), ks), Spine(x, ko), A.AGG_WCOUNT))(x.batch_from_rows(ks, wa.rows())),
          em.aggregate_delta(wa, wa, Z(ko), A.AGG_WCOUNT), "aggregate WCOUNT")
    k3, k3o = Schema("uiu"), Schema("ui", "ii")
    w2 = em.weigh(za, _expr(lval(0)), capi.WEIGH_AVG)
    check(be, ref, lambda x: (lambda d: x.aggregate_delta(d, tr_of(x, w2.rows(), k3), Spine(x, k3o), A.AGG_WCOUNT2))(x.batch_from_rows(k3, w2.rows())),
          em.aggregate_delta(w2, w2, Z(k3o), A.AGG_WCOUNT2), "aggregate WCOUNT2")
    s7 = Schema("uuuuuuu")
    r7 = rows_of(rng, s7, 50, 3)
    check(be, ref, lambda x: x.weigh(x.batch_from_rows(s7, r7), key(6), capi.WEIGH_AVG), em.weigh(Z(s7, r7), _expr(key(6)), capi.WEIGH_AVG),
          "WEIGH_AVG of 7 key lanes: 8 out")
    still_usable(be, ref, "operand-pair refusals")


# ---- sizes -------------------------------------------------------------------------------------------------------------
def run_sizes(be, ref=None):
    rng = np.random.default_rng(9)
    o = out()
    s = Schema("u", "uu")
    rows = rows_of(rng, s, 700, 200)
    z = Z(s, rows)
    b = be.batch_from_rows(s, rows)
    one = np.array([7], dtype=np.uint64)
    w1 = np.array([1], dtype=np.int64)
    cols9 = col_ptrs([one] * 9)
    p = Proj(Schema("u"), [lval(0)])
    for ncols in (0, 9, 1 << 31):
        refused(be, "batch_from_table", be.ctx, cols9, ncols, w1.ctypes.data, 1, 0, p.c(), C.byref(o), names="n_cols", outs=[o])
        refused(be, "upload_begin", be.ctx, cols9, ncols, 0xFF, w1.ctypes.data, 1, C.byref(o), names="n_cols", outs=[o])
    empty = be.batch_empty(s)
    outs = (C.c_void_p * 66)()
    for bb in (b, empty):
        for P in (0, 65, 1 << 31):
            refused(be, "shard_partition", be.ctx, bb.h, P, outs, names="n_shards")
            assert not any(outs[i] for i in range(66))
    for nk in (4, 255, 1 << 31):
        refused(be, "batch_reindex", be.ctx, b.h, nk, C.byref(o), names="n_key_lanes", outs=[o])
    for root in (-1, 1):   # a context without a comm is a group of one
        refused(be, "gather", be.ctx, b.h, root, C.byref(o), names="root", outs=[o])
    blob = (C.c_uint8 * capi.COMM_BLOB_BYTES)()
    for rank, world, names in ((0, 0, "world"), (0, 33, "world"), (0, -1, "world"), (-1, 2, "rank"), (2, 2, "rank"), (32, 32, "rank")):
        refused(be, "comm_create", be.ctx, rank, world, 4096, blob, names=names)
    refused(be, "comm_create", be.ctx, 0, 1, 4096, None, names="blob_out")
    # row counts the 32-bit row indices of the device cannot hold: refused as unsupported before anything is read
    sc = s.c()
    for n in (0xFFFFFFFF, 1 << 32, 1 << 60):
        args = (be.ctx, C.byref(sc), col_ptrs([one] * 3), w1.ctypes.data, n, 0, C.byref(o))
        refused(be, "batch_from_tuples", *args, names="n =", status=UNSUPPORTED, outs=[o])
        refused(be, "batch_from_sorted", *args, names="n =", status=UNSUPPORTED, outs=[o])
        refused(be, "batch_from_table", be.ctx, col_ptrs([one]), 1, w1.ctypes.data, n, 0, p.c(), C.byref(o), names="n =", status=UNSUPPORTED, outs=[o])
    if be.name != "oracle":   # the oracle is one worker: it has no exchange to set up in the wrong order
        refused(be, "comm_connect", be.ctx, blob, names="comm_create")
        be.comm_create(1, 2, 4096)
        try:
            refused(be, "shard", be.ctx, b.h, C.byref(o), names=["exchange", "comm_connect"], outs=[o], call_named=False)
            refused(be, "gather", be.ctx, b.h, 2, C.byref(o), names="root", outs=[o])
        finally:
            be.comm_destroy()
        be.comm_create(31, 32, 4096)   # the last rank of the largest group
        assert be.comm_info()[:2] == (31, 32)
        be.comm_destroy()
    # accepted: 64 shards, a group of one, every split of the lanes
    for P in (1, 64):
        shards = be.shard_partition(b, P)
        assert len(shards) == P
        total = Z(s)
        for sh in shards:
            total.add(sh.rows())
        assert total.rows() == z.rows(), f"{P} shards do not partition the batch"
        if ref is not None:
            for i, (x, y) in enumerate(zip(shards, ref.shard_partition(ref.batch_from_rows(s, rows), P))):
                assert_batches_equal(x, y, f"shard {i} of {P}")
        assert all(len(e) == 0 for e in be.shard_partition(empty, P))
    check(be, ref, lambda x: x.gather(x.batch_from_rows(s, rows), 0), z, "gather to root 0 of a group of one")
    check(be, ref, lambda x: x.shard(x.batch_from_rows(s, rows)), z, "shard in a group of one")
    for nk in (0, 3):
        check(be, ref, lambda x: x.reindex(x.batch_from_rows(s, rows), nk), Z(s.reindex(nk), rows), f"reindex to {nk} key lanes")
    assert len(be.reindex(empty, 3)) == 0
    tbl = [rng.integers(0, 9, 100).astype(np.uint64) for _ in range(8)]
    p8 = Proj(Schema("u", "u"), [lval(7), lval(0)])
    check(be, ref, lambda x: x.batch_from_table(tbl, p8), em.batch_from_table(tbl, p8), "from_table with 8 columns")
    check(be, ref, lambda x: x.batch_from_table(tbl[:1], p), em.batch_from_table(tbl[:1], p), "from_table with 1 column")
    still_usable(be, ref, "size refusals")


# ---- protocol ------------------------------------------------------------------------------------------------------------
def run_protocol(be, ref=None):
    rng = np.random.default_rng(11)
    s = Schema("u", "u")
    ra, rb_ = rows_of(rng, s, 900), rows_of(rng, s, 900)
    za, zb = Z(s, ra), Z(s, rb_)
    o = out()

    def merger_story(x):
        """done() before completion is refused and leaves the merger where it was; work() with no fuel or negative
        fuel does nothing: the fuel comes back unchanged (<= 0: not complete) and the merge continues from there."""
        m = x.merger(x.batch_from_rows(s, ra), x.batch_from_rows(s, rb_))
        if x is be:
            refused(be, "merger_done", be.ctx, m.h, C.byref(o), names=["merger", "not complete"], outs=[o])
        assert m.work(100) <= 0
        for fuel in (0, -1, em.MIN):
            before = counters(x)
            assert m.work(fuel) == fuel, "work() without fuel changed the fuel"
            assert counters(x) == before, "work() without fuel launched, copied or waited"
        if x is be:
            refused(be, "merger_done", be.ctx, m.h, C.byref(o), names=["merger", "not complete"], outs=[o])
        while m.work(250) <= 0:
            pass
        assert m.work(0) > 0 and m.work(-5) > 0, "a complete merge reports fuel > 0 whatever it was given"
        return m.done()

    check(be, ref, merger_story, em.union(za, zb), "fuelled merge across refused done() and fuel <= 0")
    fc, fw = em.flat(s, za)
    q = be.batcher(s)
    ptrs = col_ptrs([as_u64(c) for c in fc])
    refused(be, "batcher_push_consolidated", be.ctx, q.h, ptrs, None, len(fw), 0, names="weights is NULL")
    assert q.tuples() == 0
    sc = s.c()
    refused(be, "batch_from_sorted", be.ctx, C.byref(sc), ptrs, None, len(fw), 0, C.byref(o), names="weights is NULL", outs=[o])

    def batcher_story(x):
        qq = x.batcher(s)
        qq.push_consolidated_batch(fc, fw)
        qq.push_rows(rb_)
        return qq.seal()

    check(be, ref, batcher_story, em.union(za, zb), "push_consolidated with weights")
    cs, cw = em.consolidate_np(s, [c.copy() for c in fc], np.ones(len(fw), np.int64))
    check(be, ref, lambda x: x.batch_from_columns(s, fc, None), (cs, cw), "from_tuples without weights: all +1")
    still_usable(be, ref, "protocol refusals")


# ---- pointers --------------------------------------------------------------------------------------------------------------
def run_pointers(be, ref=None):
    s = Schema("u", "u")
    b = be.batch_from_rows(s, [(1, 2, 1), (3, 4, 1)])
    tr = Spine(be, s)
    tr.insert(b)
    sc, o, n64, i64v = s.c(), out(), C.c_uint64(), C.c_int64(5)
    one = np.array([7], dtype=np.uint64)
    cols, w1 = col_ptrs([one, one]), np.array([1], dtype=np.int64)
    p = Proj(s, [key(0), lval(0)])
    m = be.merger(b, b)
    q = be.batcher(s)
    up = be.upload_begin([one, one], 0b11, w1)
    f = _expr(lval(0)).c()
    k4 = [_lanes([0])] * 4
    api = be.api
    # a NULL context: no counters to read, so the harness's are those of the live context (they must not move either)
    null_ctx = [
        ("ctx_sync", (None,)), ("ctx_stats", (None, None, None, None, 0)), ("ctx_sync_stats", (None, None, None, 0)),
        ("batch_from_tuples", (None, C.byref(sc), cols, None, 1, 0, C.byref(o))), ("batch_from_table", (None, cols, 2, None, 1, 0, p.c(), C.byref(o))),
        ("batch_from_sorted", (None, C.byref(sc), cols, w1.ctypes.data, 1, 0, C.byref(o))), ("upload_begin", (None, cols, 2, 3, None, 1, C.byref(o))),
        ("batch_from_upload", (None, up.h, p.c(), C.byref(o))), ("batch_empty", (None, C.byref(sc), C.byref(o))),
        ("batch_merge", (None, b.h, b.h, C.byref(o))), ("batch_merge_bounded", (None, b.h, b.h, None, C.byref(o))),
        ("batcher_new", (None, C.byref(sc), C.byref(o))), ("batcher_push", (None, q.h, cols, None, 1, 0)),
        ("batcher_push_consolidated", (None, q.h, cols, w1.ctypes.data, 1, 0)), ("batcher_seal", (None, q.h, C.byref(o))),
        ("merger_new", (None, b.h, b.h, None, C.byref(o))), ("merger_work", (None, m.h, C.byref(i64v))), ("merger_done", (None, m.h, C.byref(o))),
        ("batch_truncate_keys_below", (None, b.h, _lanes([0]), C.byref(o))), ("batch_neg", (None, b.h, C.byref(o))),
        ("batch_reindex", (None, b.h, 1, C.byref(o))), ("batch_key_count", (None, b.h, C.byref(n64))),
        ("batch_download_csr", (None, b.h, None, None, None, None)), ("batch_last_key", (None, b.h, _lanes([0]), C.byref(C.c_int32()))),
        ("spine_new", (None, C.byref(sc), C.byref(o))), ("spine_insert", (None, tr.h, b.h)), ("spine_consolidate", (None, tr.h, C.byref(o))),
        ("spine_truncate_keys_below", (None, tr.h, _lanes([0]))), ("spine_truncate_values_below", (None, tr.h, _lanes([0]))),
        ("spine_exert", (None, tr.h, C.byref(i64v))), ("spine_save", (None, tr.h, b"unused")), ("spine_load", (None, b"unused", C.byref(o))),
        ("join_delta_trace", (None, b.h, tr.h, p.c(), 1, C.byref(o))), ("join_batches", (None, b.h, b.h, p.c(), C.byref(o))),
        ("semijoin", (None, b.h, b.h, C.byref(o))), ("aggregate_delta", (None, b.h, tr.h, tr.h, 0, C.byref(o))),
        ("weigh", (None, b.h, C.byref(f), 0, C.byref(o))), ("distinct_delta", (None, b.h, tr.h, C.byref(o))),
        ("stream_distinct", (None, b.h, C.byref(o))), ("window_delta", (None, tr.h, b.h, 1, *k4, C.byref(o))),
        ("map_index", (None, b.h, p.c(), C.byref(o))), ("shard_partition", (None, b.h, 1, C.byref(o))),
        ("comm_connect", (None, cols)), ("comm_destroy", (None,)), ("comm_info", (None, None, None, None)),
        ("shard", (None, b.h, C.byref(o))), ("shard2", (None, b.h, b.h, C.byref(o), C.byref(o))), ("gather", (None, b.h, 0, C.byref(o))),
        ("allreduce_max_u64", (None, C.byref(n64))),
    ]
    if be.name != "oracle":   # the oracle has neither a profile nor asynchronous reads
        null_ctx += [("ctx_profile", (None, 1)), ("ctx_profile_read", (None, 0, None, None, None, None)),
                     ("batch_download_begin", (None, b.h, None, None, C.byref(o)))]
    for call, args in null_ctx:
        refused(be, call, *args, names="ctx is NULL", outs=[o])
    refused(be, "comm_create", None, 0, 1, 0, (C.c_uint8 * capi.COMM_BLOB_BYTES)(), names="ctx is NULL")
    assert api._ctx_stream(None) is None
    assert api._ctx_destroy(None) == 0
    # NULL out-pointers, NULL inputs, NULL handles: one call or more per handle type
    for call, args, names in [
        ("ctx_create", (0, None), "out"),
        ("batch_from_tuples", (be.ctx, C.byref(sc), cols, None, 1, 0, None), "out"),
        ("batch_from_tuples", (be.ctx, None, cols, None, 1, 0, C.byref(o)), "schema is NULL"),
        ("batch_from_tuples", (be.ctx, C.byref(sc), None, None, 1, 0, C.byref(o)), "cols is NULL"),
        ("batch_from_tuples", (be.ctx, C.byref(sc), col_ptrs([one, None]), None, 1, 0, C.byref(o)), "cols[1] is NULL"),
        ("batch_from_sorted", (be.ctx, C.byref(sc), None, w1.ctypes.data, 1, 0, C.byref(o)), "cols is NULL"),
        ("batch_from_table", (be.ctx, None, 2, None, 1, 0, p.c(), C.byref(o)), "cols is NULL"),
        ("batch_from_table", (be.ctx, col_ptrs([one, None]), 2, None, 1, 0, Proj(s, [key(0), lval(1)]).c(), C.byref(o)), "cols[1] is NULL"),
        ("batch_from_table", (be.ctx, cols, 2, None, 1, 0, None, C.byref(o)), "proj is NULL"),
        ("batch_from_table", (be.ctx, cols, 2, None, 1, 0, p.c(), None), "out"),
        ("upload_begin", (be.ctx, None, 2, 3, None, 1, C.byref(o)), "cols is NULL"),
        ("upload_begin", (be.ctx, col_ptrs([one, None]), 2, 3, None, 1, C.byref(o)), "cols[1] is NULL"),
        ("upload_begin", (be.ctx, cols, 2, 3, None, 1, None), "out"),
        ("batch_from_upload", (be.ctx, None, p.c(), C.byref(o)), "upload is NULL"),
        ("batch_from_upload", (be.ctx, up.h, None, C.byref(o)), "proj is NULL"),
        ("batch_from_upload", (be.ctx, up.h, p.c(), None), "out"),
        ("batch_empty", (be.ctx, C.byref(sc), None), "out"),
        ("batch_merge", (be.ctx, None, b.h, C.byref(o)), "a is NULL"),
        ("batch_merge", (be.ctx, b.h, None, C.byref(o)), "b is NULL"),
        ("batch_merge", (be.ctx, b.h, b.h, None), "out"),
        ("batcher_new", (be.ctx, None, C.byref(o)), "schema is NULL"),
        ("batcher_push", (be.ctx, None, cols, None, 1, 0), "batcher is NULL"),
        ("batcher_push", (be.ctx, q.h, None, None, 1, 0), "cols is NULL"),
        ("batcher_push_consolidated", (be.ctx, None, cols, w1.ctypes.data, 1, 0), "batcher is NULL"),
        ("batcher_tuples", (None, C.byref(n64)), "batcher is NULL"),
        ("batcher_tuples", (q.h, None), "n_tuples"),
        ("batcher_seal", (be.ctx, None, C.byref(o)), "batcher is NULL"),
        ("batcher_seal", (be.ctx, q.h, None), "out"),
        ("merger_new", (be.ctx, None, b.h, None, C.byref(o)), "a is NULL"),
        ("merger_new", (be.ctx, b.h, b.h, None, None), "out"),
        ("merger_work", (be.ctx, None, C.byref(i64v)), "merger is NULL"),
        ("merger_work", (be.ctx, m.h, None), "fuel is NULL"),
        ("merger_done", (be.ctx, None, C.byref(o)), "merger is NULL"),
        ("merger_done", (be.ctx, m.h, None), "out"),
        ("batch_neg", (be.ctx, None, C.byref(o)), "batch is NULL"),
        ("batch_neg", (be.ctx, b.h, None), "out"),
        ("batch_reindex", (be.ctx, None, 1, C.byref(o)), "batch is NULL"),
        ("batch_len", (None, C.byref(n64)), "batch is NULL"),
        ("batch_len", (b.h, None), "n_tuples"),
        ("batch_key_count", (be.ctx, None, C.byref(n64)), "batch is NULL"),
        ("batch_key_count", (be.ctx, b.h, None), "n_keys"),
        ("batch_schema", (None, C.byref(sc)), "batch is NULL"),
        ("batch_schema", (b.h, None), "out"),
        ("batch_download_csr", (be.ctx, None, None, None, None, None), "batch is NULL"),
        ("batch_last_key", (be.ctx, b.h, None, C.byref(C.c_int32())), "key is NULL"),
        ("batch_last_key", (be.ctx, b.h, _lanes([0]), None), "valid is NULL"),
        ("batch_clone", (None, C.byref(o)), "batch is NULL"),
        ("batch_clone", (b.h, None), "out"),
        ("batch_truncate_keys_below", (be.ctx, None, _lanes([0]), C.byref(o)), "batch is NULL"),
        ("spine_new", (be.ctx, None, C.byref(o)), "schema is NULL"),
        ("spine_new", (be.ctx, C.byref(sc), None), "out"),
        ("spine_insert", (be.ctx, None, b.h), "spine is NULL"),
        ("spine_insert", (be.ctx, tr.h, None), "batch is NULL"),
        ("spine_consolidate", (be.ctx, None, C.byref(o)), "spine is NULL"),
        ("spine_consolidate", (be.ctx, tr.h, None), "out"),
        ("spine_truncate_keys_below", (be.ctx, None, _lanes([0])), "spine is NULL"),
        ("spine_truncate_values_below", (be.ctx, None, _lanes([0])), "spine is NULL"),
        ("spine_exert", (be.ctx, None, C.byref(i64v)), "spine is NULL"),
        ("spine_exert", (be.ctx, tr.h, None), "effort is NULL"),
        ("spine_len", (None, C.byref(n64), None), "spine is NULL"),
        ("spine_save", (be.ctx, None, b"unused"), "spine is NULL"),
        ("spine_save", (be.ctx, tr.h, None), "path is NULL"),
        ("spine_load", (be.ctx, None, C.byref(o)), "path is NULL"),
        ("spine_load", (be.ctx, b"unused", None), "out"),
        ("join_delta_trace", (be.ctx, None, tr.h, p.c(), 1, C.byref(o)), "delta is NULL"),
        ("join_delta_trace", (be.ctx, b.h, None, p.c(), 1, C.byref(o)), "trace is NULL"),
        ("join_delta_trace", (be.ctx, b.h, tr.h, None, 1, C.byref(o)), "proj is NULL"),
        ("join_delta_trace", (be.ctx, b.h, tr.h, p.c(), 1, None), "out"),
        ("join_batches", (be.ctx, None, b.h, p.c(), C.byref(o)), "left is NULL"),
        ("join_batches", (be.ctx, b.h, None, p.c(), C.byref(o)), "right is NULL"),
        ("semijoin", (be.ctx, None, b.h, C.byref(o)), "pairs is NULL"),
        ("semijoin", (be.ctx, b.h, None, C.byref(o)), "keys is NULL"),
        ("aggregate_delta", (be.ctx, None, tr.h, tr.h, 0, C.byref(o)), "delta is NULL"),
        ("aggregate_delta", (be.ctx, b.h, None, tr.h, 0, C.byref(o)), "in_trace is NULL"),
        ("aggregate_delta", (be.ctx, b.h, tr.h, None, 0, C.byref(o)), "out_trace is NULL"),
        ("aggregate_delta", (be.ctx, b.h, tr.h, tr.h, 0, None), "out"),
        ("weigh", (be.ctx, None, C.byref(f), 0, C.byref(o)), "batch is NULL"),
        ("distinct_delta", (be.ctx, None, tr.h, C.byref(o)), "delta is NULL"),
        ("distinct_delta", (be.ctx, b.h, None, C.byref(o)), "delayed_integral is NULL"),
        ("stream_distinct", (be.ctx, None, C.byref(o)), "batch is NULL"),
        ("window_delta", (be.ctx, None, b.h, 1, *k4, C.byref(o)), "trace is NULL"),
        ("window_delta", (be.ctx, tr.h, None, 1, *k4, C.byref(o)), "delta is NULL"),
        ("window_delta", (be.ctx, tr.h, b.h, 1, *k4, None), "out"),
        ("map_index", (be.ctx, None, p.c(), C.byref(o)), "batch is NULL"),
        ("map_index", (be.ctx, b.h, None, C.byref(o)), "proj is NULL"),
        ("map_index", (be.ctx, b.h, p.c(), None), "out"),
        ("shard_partition", (be.ctx, None, 1, C.byref(o)), "batch is NULL"),
        ("shard_partition", (be.ctx, b.h, 1, None), "outs is NULL"),
        ("comm_connect", (be.ctx, None), "blobs is NULL"),
        ("shard", (be.ctx, None, C.byref(o)), "batch is NULL"),
        ("shard", (be.ctx, b.h, None), "out"),
        ("shard2", (be.ctx, b.h, None, C.byref(o), C.byref(o)), "b is NULL"),
        ("shard2", (be.ctx, b.h, b.h, C.byref(o), None), "out_b"),
        ("gather", (be.ctx, None, 0, C.byref(o)), "batch is NULL"),
        ("gather", (be.ctx, b.h, 0, None), "out"),
        ("allreduce_max_u64", (be.ctx, None), "x is NULL"),
    ]:
        refused(be, call, *args, names=names, outs=[o])
    if be.name != "oracle":
        refused(be, "batch_download_begin", be.ctx, None, None, None, C.byref(o), names="batch is NULL", outs=[o])
        refused(be, "batch_download_begin", be.ctx, b.h, None, None, None, names="out")
        refused(be, "batch_device_columns", None, cols, None, names="batch is NULL")
        refused(be, "batch_device_columns", b.h, None, None, names="cols is NULL")
    # every *_free (and download_finish) is a no-op on NULL
    for call in ("batch_free", "spine_free", "merger_free", "batcher_free", "upload_free", "download_finish"):
        assert getattr(api, "_" + call)(None) == 0, call
    # the handles the refused calls were given are intact
    assert b.rows() == [(1, 2, 1), (3, 4, 1)] and signed_rows(tr.consolidate()) == [(1, 2, 1), (3, 4, 1)]
    assert q.tuples() == 0 and len(q.seal()) == 0
    while m.work(100) <= 0:
        pass
    assert m.done().rows() == [(1, 2, 2), (3, 4, 2)]
    em.assert_batch_is(be.batch_from_upload(up, p), Z(s, [(7, 7, 1)]), "the upload survives the refusals")
    still_usable(be, ref, "pointer refusals")


# ---- snapshot files ----------------------------------------------------------------------------------------------------------
# The format of dbsp_spine_save (include/dbsp_b200.h), little endian: magic[8] | n_key_lanes u8, n_val_lanes u8,
# lane_types[8] | has_bound, has_vbound, effort, n_layers (u64 each) | bound[8] u64 | vbound[8] u64 | per layer:
# kind u64, remaining i64, then batches a and b: present u64, n u64, L lanes of n u64, n i64 weights.
MAGIC = b"DBSPSPN1"
KINDS = {"VACANT": 0, "SINGLE": 1, "IN_PROGRESS": 2, "COMPLETE": 3}


def parse_snapshot(data):
    """(snapshot as a dict, field boundaries as (offset, what the field before it was), offsets of the middle of a lane)."""
    at, cuts, mids = 0, [], []

    def take(fmt, what):
        nonlocal at
        v = struct.unpack_from("<" + fmt, data, at)
        at += struct.calcsize("<" + fmt)
        cuts.append((at, what))
        return v

    snap = {"magic": take("8s", "magic")[0]}
    snap["nk"], snap["nv"] = take("B", "n_key_lanes")[0], take("B", "n_val_lanes")[0]
    snap["types"] = list(take("8B", "lane_types"))
    for f in ("has_bound", "has_vbound", "effort", "n_layers"):
        snap[f] = take("Q", f)[0]
    snap["bound"], snap["vbound"] = list(take("8Q", "bound")), list(take("8Q", "vbound"))
    L = snap["nk"] + snap["nv"]
    snap["layers"] = []
    for _ in range(snap["n_layers"]):
        layer = {"kind": take("Q", "kind")[0], "remaining": take("q", "remaining")[0], "batches": []}
        for which in "ab":
            bt = {"present": take("Q", f"present {which}")[0], "n": take("Q", f"n {which}")[0], "lanes": [], "w": []}
            for l in range(L + 1 if bt["n"] else 0):
                if bt["n"] > 1:
                    mids.append(at + 8 * (bt["n"] // 2))
                vals = list(take(f"{bt['n']}{'Q' if l < L else 'q'}", f"lane {l} of {which}" if l < L else f"weights of {which}"))
                if l < L:
                    bt["lanes"].append(vals)
                else:
                    bt["w"] = vals
            layer["batches"].append(bt)
        snap["layers"].append(layer)
    assert at == len(data), "the parser does not cover the whole file"
    return snap, cuts, mids


def write_snapshot(snap):
    parts = [struct.pack("<8sBB8B", snap["magic"], snap["nk"], snap["nv"], *snap["types"]),
             struct.pack("<4Q", snap["has_bound"], snap["has_vbound"], snap["effort"], snap["n_layers"]),
             struct.pack("<8Q", *snap["bound"]), struct.pack("<8Q", *snap["vbound"])]
    for layer in snap["layers"]:
        parts.append(struct.pack("<Qq", layer["kind"], layer["remaining"]))
        for bt in layer["batches"]:
            parts.append(struct.pack("<QQ", bt["present"], bt["n"]))
            for lane in bt["lanes"]:
                parts.append(struct.pack(f"<{len(lane)}Q", *lane))
            parts.append(struct.pack(f"<{len(bt['w'])}q", *bt["w"]))
    return b"".join(parts)


def snapshot_damages(snap):
    """(what, mutation of the parsed snapshot, text the refusal must contain, whether the header alone gives it away)."""
    layers = snap["layers"]
    first = lambda kind: next(i for i, l in enumerate(layers) if l["kind"] == KINDS[kind])
    single = next(i for i, l in enumerate(layers) if l["kind"] == KINDS["SINGLE"] and l["batches"][0]["n"] >= 3)
    prog = first("IN_PROGRESS")
    vac = first("VACANT")
    plen = sum(bt["n"] for bt in layers[prog]["batches"])
    L = snap["nk"] + snap["nv"]

    def setf(name, v):
        return lambda s: s.__setitem__(name, v)

    def layer(i, name, v):
        return lambda s: s["layers"][i].__setitem__(name, v)

    def batch(i, w, name, v):
        return lambda s: s["layers"][i]["batches"][w].__setitem__(name, v)

    def drop_batch(i, w):
        return lambda s: s["layers"][i]["batches"].__setitem__(w, {"present": 0, "n": 0, "lanes": [], "w": []})

    def give_batch(i):
        return lambda s: s["layers"][i]["batches"].__setitem__(0, dict(s["layers"][single]["batches"][0]))

    def swap_rows(s):
        bt = s["layers"][single]["batches"][0]
        for lane in bt["lanes"]:
            lane[0], lane[1] = lane[1], lane[0]

    def duplicate_row(s):
        bt = s["layers"][single]["batches"][0]
        for lane in bt["lanes"]:
            lane[1] = lane[0]

    def zero_weight(s):
        s["layers"][single]["batches"][0]["w"][1] = 0

    return [
        ("magic", setf("magic", b"DBSPSPN2"), "magic", True),
        ("no lanes", lambda s: (setf("nk", 0)(s), setf("nv", 0)(s)), "1..8 lanes", True),
        ("nine lanes", lambda s: (setf("nk", 5)(s), setf("nv", 4)(s)), "1..8 lanes", True),
        ("lane count wrapping uint8", lambda s: (setf("nk", 255)(s), setf("nv", L - 255 + 256)(s)), "1..8 lanes", True),
        ("lane type 2", lambda s: s["types"].__setitem__(0, 2), "lane_types[0]", True),
        ("key bound flag 2", setf("has_bound", 2), "bound flag", True),
        ("value bound flag 2", setf("has_vbound", 2), "bound flag", True),
        ("65 layers", setf("n_layers", 65), "layer count", True),
        ("kind 4", layer(0, "kind", 4), "layer kind", False),
        ("remaining -1", layer(prog, "remaining", -1), "remaining", False),
        ("remaining len + 1", layer(prog, "remaining", plen + 1), "remaining", False),
        ("presence 2", batch(single, 0, "present", 2), "presence", False),
        ("n = 2^32", batch(single, 0, "n", 1 << 32), "2^32", False),
        ("n = 2^60", batch(single, 0, "n", 1 << 60), "2^32", False),
        ("n = 2^31: more rows than the file holds", batch(single, 0, "n", 1 << 31), "does not fit", False),
        ("merge in progress without a", drop_batch(prog, 0), "without batch a", False),
        ("merge in progress without b", drop_batch(prog, 1), "without batch b", False),
        ("vacant layer with a batch", give_batch(vac), "cannot hold batch a", False),
        ("single layer with b", lambda s: s["layers"][single]["batches"].__setitem__(1, dict(s["layers"][single]["batches"][0])), "cannot hold batch b", False),
        ("absent batch with rows", lambda s: s["layers"][vac]["batches"][0].__setitem__("n", 3), "absent batch", False),
        ("two rows swapped", swap_rows, "(1 out of order", False),
        ("a row duplicated", duplicate_row, " 1 duplicates", False),
        ("a weight of 0", zero_weight, " 1 zero weights", False),
    ]


def load_refused(be, ref, path, data, names, header_only, what):
    with open(path, "wb") as f:
        f.write(data)
    o = out()
    msg = refused(be, "spine_load", be.ctx, path.encode(), C.byref(o), names=names, outs=[o], ran_nothing=header_only)
    if ref is not None:   # both libraries refuse the same file for the same reason
        assert refused(ref, "spine_load", ref.ctx, path.encode(), C.byref(o), names=names, outs=[o], ran_nothing=header_only) == msg, what


def run_snapshot_refusals(be, tmpdir, ref=None):
    import copy

    s = Schema("u", "u")
    tr, _ = snapshot_cases.build_spine(be, s, 21)
    good = os.path.join(str(tmpdir), f"good_{be.name}.bin")
    bad = os.path.join(str(tmpdir), f"bad_{be.name}.bin")
    tr.save(good)
    data = open(good, "rb").read()
    snap, cuts, mids = parse_snapshot(data)
    assert write_snapshot(snap) == data, "the test's writer does not reproduce the library's file byte for byte"
    kinds = {l["kind"] for l in snap["layers"]}
    assert {KINDS["VACANT"], KINDS["SINGLE"], KINDS["IN_PROGRESS"]} <= kinds and snap["has_bound"] == 1 and snap["has_vbound"] == 1
    want = signed_rows(tr.consolidate())
    # cut at every field boundary (the last boundary is the whole file) and in the middle of lanes
    for at, what in cuts[:-1]:
        load_refused(be, ref, bad, data[:at], "magic" if at < 8 else "truncated", at <= cuts[9][0], f"cut after {what}")
    load_refused(be, ref, bad, b"", "magic", True, "empty file")
    load_refused(be, ref, bad, data[:3], "magic", True, "cut inside the magic")
    for at in mids[:: max(1, len(mids) // 12)] + [len(data) - 1]:
        load_refused(be, ref, bad, data[:at], "truncated", False, f"cut at {at}, inside a lane")
    load_refused(be, ref, bad, data + bytes(8), "trailing", False, "8 trailing bytes")
    load_refused(be, ref, bad, data + b"\x01", "trailing", False, "1 trailing byte")
    for what, damage, names, header_only in snapshot_damages(snap):
        d = copy.deepcopy(snap)
        damage(d)
        load_refused(be, ref, bad, write_snapshot(d), names, header_only, what)
    # accepted: the file itself, re-serialised; and the nearest legal values of the fields above
    for what, edit in (("as written", lambda d: None),
                       ("remaining 0 and remaining = len", lambda d: [l.__setitem__("remaining", 0 if i % 2 else sum(b["n"] for b in l["batches"]))
                                                                      for i, l in enumerate(d["layers"]) if l["kind"] == KINDS["IN_PROGRESS"]]),
                       ("64 layers", lambda d: (d["layers"].extend(copy.deepcopy({"kind": 0, "remaining": 0, "batches": [{"present": 0, "n": 0, "lanes": [], "w": []}] * 2})
                                                                   for _ in range(64 - len(d["layers"]))), d.__setitem__("n_layers", 64)))):
        d = copy.deepcopy(snap)
        edit(d)
        with open(bad, "wb") as f:
            f.write(write_snapshot(d))
        back = Spine.load(be, bad, s)
        assert signed_rows(back.consolidate()) == want, f"accepted snapshot: {what}"
        if ref is not None:
            assert signed_rows(Spine.load(ref, bad, s).consolidate()) == want, f"accepted snapshot in the second library: {what}"
    still_usable(be, ref, "snapshot refusals")


def run_snapshot_accepts(be, tmpdir, ref=None):
    """What a trace can legitimately look like when it is saved: every row width, an empty trace, a trace whose
    layers hold only empty batches, the layers exert leaves."""
    path = os.path.join(str(tmpdir), f"ok_{be.name}.bin")
    rng = np.random.default_rng(13)
    for s in SCHEMAS:
        tr, model = Spine(be, s), Z(s)
        for n in (300, 40, 45, 1, 7):
            rows = rows_of(rng, s, n, 1 << 62)
            tr.insert(be.batch_from_rows(s, rows))
            model.add(rows)
        tr.save(path)
        back = Spine.load(be, path, s)
        assert back.stats() == tr.stats()
        em.assert_batch_is(back.consolidate(), model, f"snapshot round trip {sid(s)}")
        if ref is not None:
            em.assert_batch_is(Spine.load(ref, path, s).consolidate(), model, f"snapshot of {sid(s)} loaded by the second library")
    s = Schema("i", "u")
    empty = Spine(be, s)
    empty.save(path)
    assert Spine.load(be, path, s).stats() == (0, 0) and parse_snapshot(open(path, "rb").read())[0]["n_layers"] == 0
    # rows and their negation: once the merges are paid for, the layers hold empty batches only
    rows = rows_of(rng, s, 500)
    tr = Spine(be, s)
    b = be.batch_from_rows(s, rows)
    tr.insert(b)
    tr.insert(be.neg(b))
    tr.exert(1 << 40)
    tr.save(path)
    snap = parse_snapshot(open(path, "rb").read())[0]
    assert all(bt["n"] == 0 for l in snap["layers"] for bt in l["batches"]) and any(bt["present"] for l in snap["layers"] for bt in l["batches"])
    back = Spine.load(be, path, s)
    assert back.stats() == tr.stats() == (0, 0)
    for sp in (tr, back):   # and both go on identically
        sp.insert(be.batch_from_rows(s, rows[:100]))
    assert signed_rows(back.consolidate()) == signed_rows(tr.consolidate()) == Z(s, rows[:100]).rows()
    # exert on a trace of single layers rolls the small layers up around a structurally empty batch: whatever layer
    # states that leaves load again
    tr = Spine(be, s)
    for n in (400, 30, 3):
        tr.insert(be.batch_from_rows(s, rows_of(rng, s, n, 1 << 20)))
    tr.exert(64)
    tr.save(path)
    back = Spine.load(be, path, s)
    assert back.stats() == tr.stats() and signed_rows(back.consolidate()) == signed_rows(tr.consolidate())
    if ref is not None:
        assert signed_rows(Spine.load(ref, path, s).consolidate()) == signed_rows(tr.consolidate())


GROUPS = {"schema": run_schema, "proj": run_proj, "pairs": run_pairs, "sizes": run_sizes, "protocol": run_protocol,
          "pointers": run_pointers}
