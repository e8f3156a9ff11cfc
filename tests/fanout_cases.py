"""Backend-generic tests of fan-outs (`dbsp_*_fanout`: one row function run n_out times per input row; DESIGN §1-2).

The model: for every input row and every j in 0 .. n_out-1, evaluate the closure with fanout_index() = j (the trees
with j substituted as a constant, or a raw program on the stack machine of rowfn_cases.py), keep the row when the
filter holds, with the input row's weight, then consolidate.  It shares no code with either library.  Every case
compares a backend's batches with the model and, given a second backend (`ref`, the row-function oracle when the CUDA
library is under test), with that backend bit for bit."""
import ctypes as C

import numpy as np

import exact_model as em
from dbsp_b200 import Proj, RootCircuit, Schema, capi, col, const, fanout_index, key, val, where_
from dbsp_b200._capi import col_ptrs
from dbsp_b200.zset import Expr, Fn, Pred, Src, _fn
from edge_cases import check, edge_weights, full_lane
from exact_model import UMAX, Z, w64
from refusal_cases import out, refused
from rowfn_cases import POOL, Program, _bad, _set, bid, fn_oracle, m_project, random_program  # noqa: F401

UNSUPPORTED = 4
j = fanout_index()


# ---- the model -------------------------------------------------------------------------------------------------------
def subst(x, jv):
    """the tree with fanout_index() replaced by the constant jv"""
    if isinstance(x, Src):
        return const(jv) if x.kind == capi.SRC_FANOUT else x
    if isinstance(x, Expr):
        return Expr(x.op, subst(x.a, jv), subst(x.b, jv))
    if isinstance(x, Pred):
        return Pred(x.cmp, subst(x.a, jv), subst(x.b, jv), x.is_signed)
    f = Fn.__new__(Fn)
    f.op, f.args, f.is_bool = x.op, [subst(a, jv) for a in x.args], x.is_bool
    return f


class _Run:
    """The closure of one run j, as the model of rowfn_cases evaluates it."""

    def __init__(self, proj, jv):
        self.schema, self.jv = proj.schema, jv
        if getattr(proj, "code", None) is not None:
            self.code = proj.code
        else:
            self.code, self.out, self.where = None, [subst(o, jv) for o in proj.out], [subst(w, jv) for w in proj.where]


def _runs(proj):
    return [_Run(proj, jv) for jv in range(proj.fanout)]


def _project(run, env):
    return m_project(run, env + (None, (run.jv,)))   # a raw program's PUSH of kind 4 reads env[4][0] = j


def m_fan_table(cols, proj, weights=None):
    out, runs = Z(proj.schema), _runs(proj)
    cl = [[int(x) for x in np.asarray(c).view(np.uint64)] for c in cols]
    for i in range(len(cl[0]) if cl else 0):
        row = tuple(c[i] for c in cl)
        for r in runs:
            o = _project(r, (row, row, row))
            if o is not None:
                out.add([o + (1 if weights is None else int(weights[i]),)])
    return out


def m_fan_map(z, proj):
    out, nk, runs = Z(proj.schema), z.schema.nk, _runs(proj)
    for t, w in z.d.items():
        for r in runs:
            o = _project(r, (t[:nk], t[nk:], t[nk:]))
            if o is not None:
                out.add([o + (w,)])
    return out


class FanProgram(Program):
    """A raw program run as a fan-out."""

    is_fanout = True

    def __init__(self, schema, code, fanout):
        super().__init__(schema, code)
        self.fanout = fanout


# ---- n_out in {1, 2, 5, 64}: keep flags that drop every row, none, and a j-dependent subset -----------------------
N_OUTS = [1, 2, 5, 64]


def closures(n_out):
    lanes = [col(0) ^ (j * 0x9E3779B97F4A7C15), col(1) + j]
    return {
        "none": Proj(Schema("u", "i"), lanes, fanout=n_out),
        "all": Proj(Schema("u", "i"), lanes, where=[j.gt(n_out)], fanout=n_out),
        "subset": Proj(Schema("u", "i"), [lanes[0], (col(1) * j) % 1000],
                       where=[((col(0) >> (j % 64)) & 1).eq(1) | (col(1) + j).remu(3).eq(0)], fanout=n_out),
    }


def run_n_outs(be, ref=None, n=700):
    """Full-range lanes, weights that wrap, every keep-flag shape, on the table and the batch entry points."""
    rng = np.random.default_rng(21)
    for n_out in N_OUTS:
        rows = max(n // n_out, 20)
        cols = [full_lane(rng, "u", rows), full_lane(rng, "i", rows)]
        w = edge_weights(rng, rows)
        for name, p in closures(n_out).items():
            assert p.is_fanout and _fn("map_index", p) == "map_index_fanout"
            got = check(be, ref, lambda b: b.batch_from_table(cols, p, weights=w), m_fan_table(cols, p, w),
                        f"table n_out={n_out} {name}")
            if name == "all":
                assert len(got) == 0
            if name == "none" and n_out > 1:
                assert len(got) > rows
            s = Schema("", "ui")   # key-less: col(l) = val(l) names the same lanes as on the table
            zrows = [(int(a), int(w64(int(b))), int(c)) for a, b, c in zip(cols[0], cols[1], w)]
            check(be, ref, lambda b: b.map_index(b.batch_from_rows(s, zrows), p), m_fan_map(Z(s, zrows), p),
                  f"batch n_out={n_out} {name}")


# ---- every entry point, sizes around the 1024-row projection tile and around it / n_out ------------------------------
def sizes(n_out):
    t = 1024 // n_out
    return sorted({0, 1, t - 1, t, t + 1, 1023, 1024, 1025})


def run_entry_points(be, ref=None):
    """batch (map_index), host table, device table and upload, for n_out 2 and 5."""
    import torch

    rng = np.random.default_rng(22)
    for n_out in (2, 5):
        p = Proj(Schema("uu", "u"), [col(2) % 97, j, col(0) - j * col(1)], where=[(col(1) ^ j) & 1], fanout=n_out)
        for n in sizes(n_out):
            cols = [full_lane(rng, "u", n) for _ in range(3)]
            w = edge_weights(rng, n)
            check(be, ref, lambda b: b.batch_from_table(cols, p, weights=w), m_fan_table(cols, p, w), f"host table n_out={n_out} n={n}")
            keep = {}

            def from_device(b):
                dev = "cuda" if b.name == "cuda" else "cpu"
                ts = [torch.from_numpy(c.view(np.int64)).to(dev) for c in cols] + [torch.from_numpy(w).to(dev)]
                keep[b.name] = ts
                got = b.batch_from_table([t.data_ptr() for t in ts[:3]], p, weights=ts[3].data_ptr(), n=n, on_device=True)
                b.sync()
                return got

            check(be, ref, from_device, m_fan_table(cols, p, w), f"device table n_out={n_out} n={n}")

            def from_upload(b):
                up = b.upload_begin([c.copy() for c in cols], col_mask=b.proj_table_mask(p), weights=w)
                return b.batch_from_upload(up, p)

            check(be, ref, from_upload, m_fan_table(cols, p, w), f"upload n_out={n_out} n={n}")
            s = Schema("", "uuu")
            zrows = [tuple(int(c[i]) for c in cols) + (int(w[i]),) for i in range(n)]
            check(be, ref, lambda b: b.map_index(b.batch_from_rows(s, zrows), p), m_fan_map(Z(s, zrows), p),
                  f"batch n_out={n_out} n={n}")
    # a narrow fan-out reads one column: the upload carries only it
    narrow = Proj(Schema("u"), [col(2) + j], fanout=3)
    assert be.proj_table_mask(narrow) == 0b100 and be.api._rowfn_table_mask(narrow.c()) == 0
    cols = [full_lane(rng, "u", 300) for _ in range(3)]
    check(be, ref, lambda b: b.batch_from_upload(b.upload_begin([c.copy() for c in cols], col_mask=0b100), narrow),
          m_fan_table(cols, narrow), "upload of one column")


# ---- seeded random programs that read j ------------------------------------------------------------------------------
def run_random_programs(be, ref=None, n_programs=40, n=150):
    rng = np.random.default_rng(23)
    s = Schema("uu", "uu")
    made = 0
    while made < n_programs:
        n_out = int(rng.integers(1, 5))
        code = random_program(rng, n_out, 2, int(rng.choice([8, 16, 32, 64])))
        if code is None:
            continue
        pushes = [i for i, c in enumerate(code) if c[0] == capi.FN_PUSH and c[1] != capi.SRC_CONST]
        if not pushes:
            continue
        for i in pushes:
            if i == pushes[0] or rng.random() < 0.3:
                code[i] = (capi.FN_PUSH, capi.SRC_FANOUT, 0, 0)
        made += 1
        p = FanProgram(Schema("u" * n_out), code, int(rng.choice([1, 2, 3, 7])))
        rows = [tuple(int(rng.choice(POOL)) if rng.random() < 0.5 else int(rng.integers(0, UMAX, dtype=np.uint64, endpoint=True))
                      for _ in range(4)) + (int(rng.integers(-2, 3)),) for _ in range(n)]
        check(be, ref, lambda b: b.map_index(b.batch_from_rows(s, rows), p), m_fan_map(Z(s, rows), p),
              f"random program {made} (n_out {p.fanout}): {code}")


# ---- the reference's test_shard data (operator/communication/shard.rs:269-275) ---------------------------------------
SHARD_TUPLES = [t for n in range(1000) for t in (((n, n), 1), ((n, 1000 * n), 1))]


def run_shard_data(be):
    """`(0..1000).flat_map(|n| vec![((n, n), 1), ((n, 1000 * n), 1)])` as a two-way fan-out, from a table and from a
    batch through Stream.flat_map_index: the OrdIndexedZSet of the literal tuple list."""
    want = Z(Schema("u", "u"), [(k, v, w) for (k, v), w in SHARD_TUPLES])
    p = Proj(Schema("u", "u"), [key(0), where_(j, key(0) * 1000, key(0))], fanout=2)
    pt = Proj(Schema("u", "u"), [col(0), where_(j, col(0) * 1000, col(0))], fanout=2)
    ns = np.arange(1000, dtype=np.uint64)
    c = RootCircuit(be)
    tbl, h = c.add_input_table(1)
    from_table = tbl.flat_map_index(pt).output()
    from_batch = c.add_source(lambda: be.batch_from_columns(Schema("u"), [ns]), Schema("u")).flat_map_index(p).output()
    h.set([ns])
    c.step()
    for o in (from_table, from_batch):
        assert em.of_batch(o.value).d == want.d
        assert o.value.rows()[:3] == [(0, 0, 2), (1, 1, 1), (1, 1000, 1)]


# ---- fanout == 1 without j is the plain closure -------------------------------------------------------------------
def run_fanout_one(be):
    """Same bytes, same entry point and same batches as the Proj without a fan-out, for both closure forms."""
    rng = np.random.default_rng(24)
    cols = [full_lane(rng, "u", 2000), full_lane(rng, "u", 2000)]
    for out_, where in (([col(0), col(1) - 3], [col(1).lt(col(0))]), ([col(0) % 7, col(1) >> 3], [(col(0) ^ col(1)) & 1])):
        plain, one = Proj(Schema("u", "u"), out_, where), Proj(Schema("u", "u"), out_, where, fanout=1)
        assert not one.is_fanout and one.is_fn == plain.is_fn and bytes(one._c) == bytes(plain._c)
        for call in ("batch_from_table", "batch_from_upload", "map_index"):
            assert _fn(call, one) == _fn(call, plain)
        a, b = be.batch_from_table(cols, plain), be.batch_from_table(cols, one)
        assert a == b and len(a) > 0
        rows = be.reindex(a, 0)   # key-less: col(l) names lane l
        assert be.map_index(rows, plain) == be.map_index(rows, one)


# ---- refusals: one per new rule --------------------------------------------------------------------------------------
def run_refusals(be, ref=None):
    s = Schema("u", "uu")
    rows = [(1, 2, 3, 1), (4, 5, 6, -1)]
    base = be.batch_from_rows(s, rows)
    p = Proj(Schema("u", "u"), [key(0) + j, val(1)], fanout=2)
    o = out()
    for n_out in (0, capi.MAX_FANOUT + 1):
        refused(be, "map_index_fanout", be.ctx, base.h, p.c(), n_out, C.byref(o), names=[f"n_out = {n_out}", "1..64"], outs=[o])
    a = np.array([1, 2], np.uint64)
    refused(be, "batch_from_table_fanout", be.ctx, col_ptrs([a]), 1, None, 2, 0, Proj(Schema("u"), [col(0) + j], fanout=2).c(), 0,
            C.byref(o), names=["n_out = 0"], outs=[o])
    # n * n_out >= 2^32: refused from the sizes; the two columns are never read
    for n, n_out in ((1 << 26, 64), ((1 << 31) + 1, 2), (0xFFFFFFFE, 2)):
        refused(be, "batch_from_table_fanout", be.ctx, col_ptrs([a]), 1, None, n, 0, Proj(Schema("u"), [col(0) + j], fanout=n_out).c(),
                n_out, C.byref(o), names=["n * n_out", "2^32-1"], status=UNSUPPORTED, outs=[o])
    # a FANOUT push anywhere but a `_fanout` call is outside the enum, with the text of any other bad kind
    refused(be, "map_index_fn", be.ctx, base.h, p.c(), C.byref(o), names=["fn.code[1].kind = 4", "not a source kind"], outs=[o])
    refused(be, "batch_from_table_fn", be.ctx, col_ptrs([a]), 1, None, 2, 0, Proj(Schema("u"), [col(0) + j], fanout=2).c(),
            C.byref(o), names=["fn.code[1].kind = 4", "not a source kind"], outs=[o])
    assert be.api._rowfn_table_mask(p.c()) == 0 and be.api._fanout_table_mask(p.c()) == 0b11
    assert be.api._fanout_table_mask(None) == 0
    # the rules valid_rowfn has always had still hold in the fan-out calls
    refused(be, "map_index_fanout", be.ctx, base.h, _bad(p, _set(3, idx=2)), 2, C.byref(o), names=["fn.code[3].idx = 2", "SRC_LVAL has 2 lanes"], outs=[o])
    up = be.upload_begin([a, a], col_mask=0b01)
    refused(be, "batch_from_upload_fanout", be.ctx, up.h, Proj(Schema("u"), [col(1) + j], fanout=2).c(), 2, C.byref(o),
            names=["fn reads column 1", "col_mask"], outs=[o])
    # the context is still usable: the fan-out at the n_out limit
    lim = Proj(Schema("u", "u"), [key(0) + j, val(1) * j], fanout=capi.MAX_FANOUT)
    check(be, ref, lambda b: b.map_index(b.batch_from_rows(s, rows), lim), m_fan_map(Z(s, rows), lim), "n_out = 64 after refusals")


# ---- q5 as its SQL states it (nexmark queries/q5.rs:24-60) -----------------------------------------------------------
def m_q5_hop(bids, slide=2_000, size=10_000):
    """The SQL over every bid so far: per hop window, the auctions whose bid count is the window's maximum, as
    {(auction, num): number of windows}."""
    counts = {}
    for a, _, _, dt, _ in bids:
        last = dt - dt % slide
        for s in range(last, last - size, -slide):
            if s >= 0:
                counts[(a, s)] = counts.get((a, s), 0) + 1
    maxn = {}
    for (a, s), c in counts.items():
        maxn[s] = max(maxn.get(s, 0), c)
    out = {}
    for (a, s), c in counts.items():
        if c >= maxn[s]:
            out[(a, c)] = out.get((a, c), 0) + 1
    return out


# dt < 8000 (windows that would start below 0), bids on window edges (1999 / 2000 / 9999 / 10000), ties for the max,
# and a later step that moves the max of windows the first steps filled
Q5_STEPS = [
    [bid(auction=1, date_time=0), bid(auction=1, date_time=1_999), bid(auction=2, date_time=2_000),
     bid(auction=2, date_time=3_500), bid(auction=3, date_time=7_999)],
    [bid(auction=3, date_time=8_000), bid(auction=1, date_time=9_999), bid(auction=2, date_time=10_000),
     bid(auction=4, date_time=11_999), bid(auction=4, date_time=12_000)],
    [bid(auction=4, date_time=12_001), bid(auction=4, date_time=13_000), bid(auction=5, date_time=25_000),
     bid(auction=3, date_time=2_500), bid(auction=1, date_time=1_000)],
]


def run_q5_hop(be, steps=Q5_STEPS):
    from dbsp_b200.nexmark import queries as nq

    c = RootCircuit(be)
    inp, handles = nq.add_nexmark_input(c)
    q = nq.QUERIES["q5_hop"](inp)
    seen = []
    q.integrate().inspect(lambda b: seen.append(em.of_batch(b)))
    bids = []
    for step in steps:
        for k in ("person", "auction"):
            handles[k].set([np.zeros(0, np.uint64)] * 5)
        handles["bid"].set([np.array(x, np.uint64) for x in zip(*step)])
        c.step()
        bids += step
        want = m_q5_hop(bids)
        got = dict(seen[-1].d)
        assert got == want, (len(bids), got, want)
    return seen[-1]
