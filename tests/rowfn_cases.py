"""Backend-generic tests of row functions (`dbsp_rowfn`, the closure form for expression trees; DESIGN §1-2).

The model here evaluates expression trees and postfix programs in Python ints; it shares no code with either library
and none with the trees' compiler in zset.py (it walks the trees the tests build, or the instruction array of a
program).  Every case compares a backend's batches with the model and, given a second backend (`ref`, the oracle when
the CUDA library is under test), with that backend bit for bit."""
import ctypes as C

import numpy as np

import exact_model as em
from dbsp_b200 import Proj, RootCircuit, Schema, Spine, capi, col, const, key, lval, rval, val, where_
from dbsp_b200._capi import CRowFn, col_ptrs
from dbsp_b200.zset import Expr, Fn, Pred, Src
from edge_cases import I_POOL, U_POOL, check
from exact_model import UMAX, Z, u64, w64
from parity_util import run_nexmark_pair
from refusal_cases import out, refused

def fn_oracle():
    """The CPU oracle with row functions (oracle_fn/libdbsp_oracle_fn.so), rebuilt when its sources are newer."""
    import __graft_entry__ as ge
    from oracle_backend import OracleBackend

    return OracleBackend(ge.build_oracle_fn())


# ---- the model -------------------------------------------------------------------------------------------------------
def _div(a, b):
    sa, sb = w64(a), w64(b)
    if sb == 0:
        return 0
    q = abs(sa) // abs(sb)
    return u64(q if (sa < 0) == (sb < 0) else -q)


def _rem(a, b):
    sa, sb = w64(a), w64(b)
    if sb == 0:
        return 0
    return u64(sa - w64(_div(a, b)) * sb)   # sign of the dividend; MIN % -1 = 0


BIN = {
    capi.FN_ADD: lambda a, b: u64(a + b), capi.FN_SUB: lambda a, b: u64(a - b), capi.FN_MUL: lambda a, b: u64(a * b),
    capi.FN_DIV: _div, capi.FN_REM: _rem,
    capi.FN_DIVU: lambda a, b: a // b if b else 0, capi.FN_REMU: lambda a, b: a % b if b else 0,
    capi.FN_MIN: lambda a, b: a if w64(a) <= w64(b) else b, capi.FN_MAX: lambda a, b: a if w64(a) >= w64(b) else b,
    capi.FN_MINU: min, capi.FN_MAXU: max,
    capi.FN_AND: lambda a, b: a & b, capi.FN_OR: lambda a, b: a | b, capi.FN_XOR: lambda a, b: a ^ b,
    capi.FN_SHL: lambda a, b: u64(a << (b % 64)), capi.FN_SHR: lambda a, b: a >> (b % 64),
    capi.FN_SAR: lambda a, b: u64(w64(a) >> (b % 64)),
    capi.FN_EQ: lambda a, b: int(a == b), capi.FN_NE: lambda a, b: int(a != b),
    capi.FN_LT: lambda a, b: int(w64(a) < w64(b)), capi.FN_LE: lambda a, b: int(w64(a) <= w64(b)),
    capi.FN_GT: lambda a, b: int(w64(a) > w64(b)), capi.FN_GE: lambda a, b: int(w64(a) >= w64(b)),
    capi.FN_LTU: lambda a, b: int(a < b), capi.FN_LEU: lambda a, b: int(a <= b),
    capi.FN_GTU: lambda a, b: int(a > b), capi.FN_GEU: lambda a, b: int(a >= b),
    capi.FN_IN: lambda a, b: int(a < 64 and (b >> a) & 1 == 1),
}
UN = {capi.FN_NEG: lambda a: u64(-a), capi.FN_ABS: lambda a: u64(abs(w64(a))), capi.FN_BNOT: lambda a: a ^ UMAX,
      capi.FN_LNOT: lambda a: int(a == 0)}


def ev(x, env):
    """u64 bit pattern of a value tree (Src / Expr / Pred / Fn) over env = (key, lval, rval) lanes."""
    if isinstance(x, Src):
        return em.src(x, env)
    if isinstance(x, Expr):
        return em.expr(x, env)
    if isinstance(x, Pred):
        a, b = ev(x.a, env), ev(x.b, env)
        if x.cmp == capi.CMP_IN:
            return BIN[capi.FN_IN](a, b)
        if x.is_signed:
            a, b = w64(a), w64(b)
        return int({capi.CMP_EQ: a == b, capi.CMP_NE: a != b, capi.CMP_LT: a < b, capi.CMP_LE: a <= b,
                    capi.CMP_GT: a > b, capi.CMP_GE: a >= b}[x.cmp])
    assert isinstance(x, Fn), x
    v = [ev(a, env) for a in x.args]
    if x.op == capi.FN_SELECT:
        return v[1] if v[0] else v[2]
    return UN[x.op](*v) if x.op in UN else BIN[x.op](*v)


def run_code(code, env):
    """The stack machine over an instruction array (ctypes CRowFn or a list of (op, kind, idx, cst))."""
    st = []
    for op, kind, idx, cst in code:
        if op == capi.FN_PUSH:
            st.append(u64(cst) if kind == capi.SRC_CONST else u64(env[kind][idx]))
        elif op == capi.FN_SELECT:
            c, a, b = st[-3:]
            del st[-3:]
            st.append(a if c else b)
        elif op in UN:
            st.append(UN[op](st.pop()))
        else:
            b = st.pop()
            st.append(BIN[op](st.pop(), b))
    return st


def m_project(proj, env):
    """The output row (typed lanes) or None: the tree form of a Proj, or its program when it carries one."""
    if getattr(proj, "code", None) is not None:
        st = run_code(proj.code, env)
        lanes, keep = st[:-1], st[-1]
    else:
        lanes, keep = [ev(o, env) for o in proj.out], all(ev(w, env) for w in proj.where)
    return tuple(em.typed(t, x) for t, x in zip(proj.schema.lanes, lanes)) if keep else None


def m_table(cols, proj, weights=None):
    out = Z(proj.schema)
    cl = [[int(x) for x in np.asarray(c).view(np.uint64)] for c in cols]
    for i in range(len(cl[0])):
        row = tuple(c[i] for c in cl)
        r = m_project(proj, (row, row, row))
        if r is not None:
            out.add([r + (1 if weights is None else int(weights[i]),)])
    return out


def m_map_index(z, proj):
    out, nk = Z(proj.schema), z.schema.nk
    for t, w in z.d.items():
        r = m_project(proj, (t[:nk], t[nk:], t[nk:]))
        if r is not None:
            out.add([r + (w,)])
    return out


def m_join(left, right, proj, swap=False):
    out, gr = Z(proj.schema), right.groups()
    for k, lvs in left.groups().items():
        for v1, w1 in lvs:
            for v2, w2 in gr.get(k, ()):
                r = m_project(proj, (k, v2, v1) if swap else (k, v1, v2))
                if r is not None:
                    out.add([r + (w1 * w2,)])
    return out


def m_weigh(z, fproj, mode):
    """weigh with a one-lane closure: a dropped row counts neither in the sum nor in the count"""
    avg = mode == capi.WEIGH_AVG
    out = Z(Schema(z.schema.key + ("u" if avg else "")))
    for k, vs in z.groups().items():
        s = c = 0
        for v, w in vs:
            r = m_project(fproj, (k, v, v))
            if r is not None:
                s, c = s + u64(r[0]) * w, c + w
        out.add([k + (0, s), k + (1, c)] if avg else [k + (s,)])
    return out


class Program:
    """A Proj-shaped wrapper of a raw program (random programs): the backends get the CRowFn, the model its code."""

    is_fn = True

    def __init__(self, schema, code):
        self.schema, self.code = schema, code
        f = CRowFn()
        f.out_schema = schema.c()
        f.n_insn = len(code)
        for i, (op, kind, idx, cst) in enumerate(code):
            f.code[i].op, f.code[i].kind, f.code[i].idx, f.code[i].cst = op, kind, idx, w64(cst)
        self._c = f

    def c(self):
        return C.byref(self._c)


# ---- every operation on the full-range pools ----------------------------------------------------------------------
POOL = sorted({u64(x) for x in U_POOL + I_POOL + [2, 3, 7, 63, 64, 123, 200, -7, -123]})
UNARY = [capi.FN_NEG, capi.FN_ABS, capi.FN_BNOT, capi.FN_LNOT]
BINARY = sorted(BIN)


def run_every_op(be, ref=None):
    """Every unary op over the pool, every binary op over all pool pairs (divisors 0 and -1, shift counts 0, 63, 64,
    200 included), SELECT over condition x pool pairs: (operands) -> result rows from a raw table."""
    a = np.array(POOL, np.uint64)
    for op in UNARY:
        p = Proj(Schema("u", "u"), [col(0), Fn(op, col(0))])
        check(be, ref, lambda b: b.batch_from_table([a], p), m_table([a], p), f"unary op {op}")
    x, y = (np.array(v, np.uint64) for v in zip(*[(i, j) for i in POOL for j in POOL]))
    for op in BINARY:
        p = Proj(Schema("uu", "u"), [col(0), col(1), Fn(op, col(0), col(1))])
        check(be, ref, lambda b: b.batch_from_table([x, y], p), m_table([x, y], p), f"binary op {op}")
    c = np.array([0, 1, 2, UMAX] * (len(x) // 4 + 1), np.uint64)[: len(x)]
    p = Proj(Schema("uuu", "u"), [col(0), col(1), col(2), where_(col(0), col(1), col(2))])
    check(be, ref, lambda b: b.batch_from_table([c, x, y], p), m_table([c, x, y], p), "select")


# ---- every entry point ----------------------------------------------------------------------------------------------
NESTED = Proj(Schema("i", "uu"), [abs(col(0) % 7 - col(1)), (col(1) * 89).divu(100), col(0).min(col(2)).signed() ^ col(1)],
              where=[(col(0) % 3).eq(0) | ~col(1).lt(1 << 63), col(2) & 1])


def u64r(rng, n=None):
    return rng.integers(0, UMAX, n, dtype=np.uint64, endpoint=True)


def table_cols(rng, n):
    return [rng.choice(np.array(POOL, np.uint64), n), u64r(rng, n), u64r(rng, n)]


def run_tables(be, ref=None, n=5000):
    """dbsp_batch_from_table_fn from host columns, device columns (torch tensors on the backend's device) and an
    upload; the columns the program reads only."""
    import torch

    rng = np.random.default_rng(11)
    cols = table_cols(rng, n)
    w = rng.integers(-3, 4, n).astype(np.int64)
    assert NESTED.is_fn and be.proj_table_mask(NESTED) == 0b111
    for wt in (None, w):
        check(be, ref, lambda b: b.batch_from_table(cols, NESTED, weights=wt), m_table(cols, NESTED, wt), f"host table w={wt is not None}")
    dev_cols = {}

    def from_device(b):
        dev = "cuda" if b.name == "cuda" else "cpu"
        ts = [torch.from_numpy(c.view(np.int64)).to(dev) for c in cols] + [torch.from_numpy(w).to(dev)]
        dev_cols[b.name] = ts   # alive until the batch is built
        got = b.batch_from_table([t.data_ptr() for t in ts[:3]], NESTED, weights=ts[3].data_ptr(), n=n, on_device=True)
        b.sync()
        return got

    check(be, ref, from_device, m_table(cols, NESTED, w), "device table")
    narrow = Proj(Schema("u"), [col(2) >> 3], where=[(col(2) & 7).ne(0)])   # reads column 2 only
    assert be.proj_table_mask(narrow) == 0b100

    def from_upload(b):
        up = b.upload_begin([c.copy() for c in cols], col_mask=be.proj_table_mask(narrow), weights=w)
        return b.batch_from_upload(up, narrow)

    check(be, ref, from_upload, m_table(cols, narrow, w), "upload")


def run_map_join_weigh(be, ref=None):
    rng = np.random.default_rng(12)
    s = Schema("u", "iu")
    rows = [(int(rng.integers(0, 40)), int(rng.choice(I_POOL)), int(rng.choice(U_POOL)), int(rng.integers(-2, 3))) for _ in range(600)]
    z = Z(s, rows)
    mi = Proj(Schema("i", "u"), [val(0) // (key(0) - 20), where_(val(0).lt(0).signed(), val(1), -val(1))],
              where=[~(key(0) % 5).eq(0)])
    check(be, ref, lambda b: b.map_index(b.batch_from_rows(s, rows), mi), m_map_index(z, mi), "map_index_fn")
    rs = Schema("u", "u")
    rrows = [(int(rng.integers(0, 40)), int(u64r(rng)), int(rng.integers(-2, 3))) for _ in range(500)]
    rz = Z(rs, rrows)
    jp = Proj(Schema("uu", "i"), [key(0), (lval(1) ^ rval(0)) >> 60, lval(0) - (rval(0) & 255)],
              where=[lval(0).gt(rval(0) % 1000).signed() | key(0).lt(5)])
    check(be, ref, lambda b: b.join_batches(b.batch_from_rows(s, rows), b.batch_from_rows(rs, rrows), jp), m_join(z, rz, jp),
          "join_batches_fn")
    for delta_is_left in (True, False):
        def jt(b):
            tr = Spine(b, rs if delta_is_left else s)
            half = len(rrows) // 2
            src = rrows if delta_is_left else rows
            sch = rs if delta_is_left else s
            tr.insert(b.batch_from_rows(sch, src[:half]))
            tr.insert(b.batch_from_rows(sch, src[half:]))
            d = b.batch_from_rows(s, rows) if delta_is_left else b.batch_from_rows(rs, rrows)
            return b.join_delta_trace(d, tr, jp, delta_is_left=delta_is_left)

        check(be, ref, jt, m_join(z, rz, jp), f"join_delta_trace_fn delta_is_left={delta_is_left}")
    f = Proj(Schema("u"), [abs(val(0)) % 1000], where=[val(1).remu(3).ne(0)])
    for mode in (capi.WEIGH_LINEAR, capi.WEIGH_AVG):
        check(be, ref, lambda b: b.weigh(b.batch_from_rows(s, rows), f, mode), m_weigh(z, f, mode), f"weigh_fn mode {mode}")
    # aggregate_linear with a filtered factor through the circuit: the per-key sum of the factor over kept rows
    c = RootCircuit(be)
    steps = [rows[:300], rows[300:]]
    it = iter([be.batch_from_rows(s, r) for r in steps])
    seen = []
    c.add_source(lambda: next(it), s).aggregate_linear(f).integrate().inspect(lambda b: seen.append(em.of_batch(b)))
    acc = Z(s)
    for r in steps:
        c.step()
        acc.add(r)
        lin = m_weigh(acc, f, capi.WEIGH_LINEAR)
        want = Z(Schema(s.key, "i"), [k + (w, 1) for k, w in lin.d.items()])
        assert seen[-1].d == want.d, "aggregate_linear with a filtered factor"


# ---- sizes around the projection's 1024-row tile --------------------------------------------------------------------
SIZES = [0, 1, 1023, 1024, 1025, 70_001]


def run_sizes(be, ref=None, sizes=SIZES):
    """A filtering program (the scan path) and one whose keep flag is the constant 1 (the identity path)."""
    rng = np.random.default_rng(13)
    keep_all = Proj(Schema("u", "u"), [col(0) % 1000, (col(1) * 3) ^ col(0)], where=[])
    assert keep_all.is_fn
    for n in sizes:
        cols = [u64r(rng, n), u64r(rng, n)]
        for p in (keep_all, NESTED_2):
            check(be, ref, lambda b: b.batch_from_table(cols, p), m_table(cols, p), f"n={n} filtered={bool(p.where)}")


NESTED_2 = Proj(Schema("u", "u"), [col(0) % 1000, col(1) >> 7], where=[(col(0) ^ col(1)) & 3])


# ---- seeded random well-formed programs ------------------------------------------------------------------------------
def random_program(rng, n_out, n_src, max_len):
    """1..max_len instructions, depth <= 16, ending at n_out + 1 values."""
    target = n_out + 1
    code, depth = [], 0
    length = int(rng.integers(target, max_len + 1))
    while len(code) < length or depth != target:
        left = max_len - len(code)
        choices = []
        if depth < capi.MAX_STACK and depth - target < left - 1:
            choices.append("push")
        if depth >= 1:
            choices.append("un")
        if depth >= 2 and depth > target - left:
            choices.append("bin")
        if depth >= 3 and depth - 1 > target - left:
            choices.append("sel")
        if depth > target and left <= depth - target:
            choices = [c for c in choices if c in ("bin", "sel")] or ["bin"]
        kind = choices[int(rng.integers(len(choices)))]
        if kind == "push":
            if rng.random() < 0.3:
                code.append((capi.FN_PUSH, capi.SRC_CONST, 0, int(rng.choice(POOL))))
            else:
                code.append((capi.FN_PUSH, int(rng.integers(0, 3)), int(rng.integers(0, n_src)), 0))
            depth += 1
        elif kind == "un":
            code.append((int(rng.choice(UNARY)), 0, 0, 0))
        elif kind == "bin":
            code.append((int(rng.choice(BINARY)), 0, 0, 0))
            depth -= 1
        else:
            code.append((capi.FN_SELECT, 0, 0, 0))
            depth -= 2
        if len(code) > max_len:
            return None
    return code


def run_random_programs(be, ref=None, n_programs=60, n=400):
    rng = np.random.default_rng(14)
    s = Schema("uu", "uu")
    made = 0
    while made < n_programs:
        n_out = int(rng.integers(1, 5))
        code = random_program(rng, n_out, 2, int(rng.choice([8, 16, 32, 64])))
        if code is None:
            continue
        made += 1
        p = Program(Schema("u" * n_out), code)
        rows = [tuple(int(rng.choice(POOL)) if rng.random() < 0.5 else int(u64r(rng)) for _ in range(4))
                + (int(rng.integers(-2, 3)),) for _ in range(n)]
        z = Z(s, rows)
        check(be, ref, lambda b: b.map_index(b.batch_from_rows(s, rows), p), m_map_index(z, p), f"random program {made}: {code}")


# ---- lowering: the Nexmark closures as programs give the same batches -----------------------------------------------
class Lowered:
    """A backend whose closure-taking calls get every closure as a row function."""

    def __init__(self, be):
        self.be, self.name = be, be.name

    def __getattr__(self, n):
        return getattr(self.be, n)

    def batch_from_table(self, cols, proj, **kw):
        return self.be.batch_from_table(cols, proj.as_rowfn(), **kw)

    def batch_from_upload(self, up, proj):
        return self.be.batch_from_upload(up, proj.as_rowfn())

    def proj_table_mask(self, proj):
        return self.be.proj_table_mask(proj.as_rowfn())

    def map_index(self, b, proj):
        return self.be.map_index(b, proj.as_rowfn())

    def join_delta_trace(self, d, tr, proj, delta_is_left=True):
        return self.be.join_delta_trace(d, tr, proj.as_rowfn(), delta_is_left)

    def join_batches(self, a, b, proj):
        return self.be.join_batches(a, b, proj.as_rowfn())

    def weigh(self, b, f, mode):
        return self.be.weigh(b, f if isinstance(f, Proj) else Proj(Schema("u"), [f]), mode)


def run_lowering(be, query, n_events=60_000, step=20_000):
    """q0 / q3 / q4 / q7 with every closure lowered to a program: step for step the batches of the dbsp_proj form."""
    return run_nexmark_pair(be, Lowered(be), query, n_events=n_events, step=step, rate=1_000)


# ---- refusals: one case per rule of valid_rowfn -----------------------------------------------------------------------
def _bad(p, fn):
    c = CRowFn.from_buffer_copy(p._c)
    fn(c)
    return C.byref(c)


def _set(i, **kw):
    def f(c):
        for k, v in kw.items():
            setattr(c.code[i], k, v)
    return f


def run_refusals(be, ref=None):
    s = Schema("u", "uu")
    base = be.batch_from_rows(s, [(1, 2, 3, 1), (4, 5, 6, -1)])
    p = Proj(Schema("u", "u"), [key(0) % 3, val(1) + val(0) * 2])   # PUSH k0, PUSH 3, REM, PUSH v1, PUSH v0, PUSH 2, MUL, ADD, PUSH 1
    assert p.is_fn and p._c.n_insn == 9
    o = out()
    cases = [
        (None, ["fn is NULL"]),
        (_bad(p, lambda c: setattr(c.out_schema, "n_key_lanes", 0) or setattr(c.out_schema, "n_val_lanes", 0)), ["fn.out_schema", "1..8 lanes"]),
        (_bad(p, lambda c: setattr(c, "n_insn", 65)), ["fn.n_insn = 65", "exceeds 64"]),
        (_bad(p, _set(2, op=34)), ["fn.code[2].op = 34", "not an instruction"]),
        (_bad(p, _set(0, kind=4)), ["fn.code[0].kind = 4", "not a source kind"]),
        (_bad(p, _set(3, idx=2)), ["fn.code[3].idx = 2", "SRC_LVAL has 2 lanes"]),
        (_bad(p, _set(0, op=capi.FN_NEG)), ["fn.code[0]", "stack underflow"]),
        (_bad(p, lambda c: setattr(c, "n_insn", 8)), ["ends with stack depth 2", "needs 3"]),
    ]
    deep = [(capi.FN_PUSH, capi.SRC_CONST, 0, 1)] * 17 + [(capi.FN_ADD, 0, 0, 0)] * 14
    cases.append((Program(Schema("u", "u"), deep).c(), ["fn.code[16]", "stack deeper than 16"]))
    for bad, names in cases:
        refused(be, "map_index_fn", be.ctx, base.h, bad, C.byref(o), names=names, outs=[o])
    # the same rules in the other entry points (the source lanes of each call)
    a = np.array([1, 2], np.uint64)
    tbl = Proj(Schema("u"), [col(1) % 2])
    refused(be, "batch_from_table_fn", be.ctx, col_ptrs([a, a]), 1, None, 2, 0, tbl.c(), C.byref(o), names=["fn.code[0].idx = 1"], outs=[o])
    up = be.upload_begin([a, a], col_mask=0b01)
    refused(be, "batch_from_upload_fn", be.ctx, up.h, tbl.c(), C.byref(o), names=["fn reads column 1", "col_mask"], outs=[o])
    jp = Proj(Schema("u"), [rval(2) % 2])
    refused(be, "join_batches_fn", be.ctx, base.h, base.h, _bad(jp, _set(0, idx=2)), C.byref(o), names=["fn.code[0].idx = 2", "SRC_RVAL has 2 lanes"], outs=[o])
    tr = Spine(be, s)
    refused(be, "join_delta_trace_fn", be.ctx, base.h, tr.h, _bad(jp, _set(0, kind=9)), 1, C.byref(o), names=["fn.code[0].kind = 9"], outs=[o])
    two = Proj(Schema("u", "u"), [key(0) % 2, val(0) % 2])
    refused(be, "weigh_fn", be.ctx, base.h, two.c(), capi.WEIGH_LINEAR, C.byref(o), names=["one lane"], outs=[o])
    assert be.api._rowfn_table_mask(None) == 0 and be.api._rowfn_table_mask(_bad(p, _set(2, op=40))) == 0
    # accepted at the limits: 64 instructions, depth 16
    limit = [(capi.FN_PUSH, capi.SRC_KEY, 0, 0)] * 16 + [(capi.FN_XOR, 0, 0, 0)] * 15 + [(capi.FN_NEG, 0, 0, 0)] * 30 + \
        [(capi.FN_PUSH, capi.SRC_LVAL, 1, 0), (capi.FN_BNOT, 0, 0, 0), (capi.FN_PUSH, capi.SRC_CONST, 0, 1)]
    lp = Program(Schema("u", "u"), limit)
    assert len(lp.code) == 64
    rows = [(1, 2, 3, 1), (4, 5, 6, -1)]
    check(be, ref, lambda b: b.map_index(b.batch_from_rows(s, rows), lp), m_map_index(Z(s, rows), lp), "64 instructions, depth 16")


# ---- the reference's literal tests -------------------------------------------------------------------------------------
# make_bid (nexmark generator/mod.rs:174-184): auction 1, bidder 1, price 99, date_time 0; extra "" = code 0
def bid(auction=1, bidder=1, price=99, date_time=0, extra=0):
    return (auction, bidder, price, date_time, extra)


Q1_STEPS = [[bid(auction=1, date_time=1_000, price=80), bid(auction=1, date_time=2_000, price=100)],
            [bid(auction=2, date_time=1_000, price=80), bid(auction=2, date_time=2_000, price=100)]]
Q2_STEPS = [[bid(auction=1, price=80), bid(auction=123, price=111), bid(auction=124, price=100)],
            [bid(auction=3 * 123 + 25, price=80), bid(auction=4 * 123, price=222)]]
Q2_OUT = [{(123, 111): 1}, {(4 * 123, 222): 1}]


def run_reference_q1_q2(be):
    """test_q1 (nexmark queries/q1.rs:43-150) and test_q2 (q2.rs:33-108) on the Nexmark input tables."""
    from dbsp_b200.nexmark import queries as nq

    for q, steps in (("q1", Q1_STEPS), ("q2", Q2_STEPS)):
        c = RootCircuit(be)
        inp, handles = nq.add_nexmark_input(c)
        o = nq.QUERIES[q](inp).output()
        for i, step in enumerate(steps):
            for k in ("person", "auction"):
                handles[k].set([np.zeros(0, np.uint64)] * 5)
            handles["bid"].set([np.array(x, np.uint64) for x in zip(*step)])
            c.step()
            got = {tuple(r[:-1]): r[-1] for r in o.value.rows()}
            if q == "q1":
                want = {(a, b, p * 89 // 100, d, e): 1 for a, b, p, d, e in step}
            else:
                want = Q2_OUT[i]
            assert got == want, (q, i, got)


# filter_map_test (operator/filter_map.rs:767-774, 799-812): the four `abs` outputs, on its literal input
ABS_INPUT = [(1, "1"), (-1, "-1"), (5, "5 foo"), (-2, "-2")]
ABS_CODE = {"-1": 0, "-2": 1, "1": 2, "5 foo": 3}
ABS_CASES = {
    "abs": ("ints", Proj(Schema("i"), [abs(key(0))]), {(1,): 2, (5,): 1, (2,): 1}),
    "abs_pos": ("ints", Proj(Schema("i"), [abs(key(0))], [key(0).gt(0).signed()]), {(1,): 1, (5,): 1}),
    "i_abs": ("indexed", Proj(Schema("iu"), [abs(key(0)), val(0)]),
              {(1, ABS_CODE["1"]): 1, (1, ABS_CODE["-1"]): 1, (5, ABS_CODE["5 foo"]): 1, (2, ABS_CODE["-2"]): 1}),
    "i_abs_pos": ("indexed", Proj(Schema("iu"), [abs(key(0)), val(0)], [key(0).gt(0).signed()]),
                  {(1, ABS_CODE["1"]): 1, (5, ABS_CODE["5 foo"]): 1}),
}


def run_abs_case(be, name):
    src, proj, want = ABS_CASES[name]
    assert proj.is_fn
    pairs = be.batch_from_rows(Schema("iu"), [(a, ABS_CODE[b], 1) for a, b in ABS_INPUT])
    indexed = be.reindex(pairs, 1)
    ints = be.map_index(indexed, Proj(Schema("i"), [key(0)]))
    got = {tuple(int(x) for x in r[:-1]): int(r[-1]) for r in be.map_index(ints if src == "ints" else indexed, proj).rows()}
    assert got == want, (name, got)


def run_dbsp_proj_bytes_unchanged():
    """A closure that fits dbsp_proj still compiles to one, byte for byte as the lanes and predicates spell it."""
    from dbsp_b200._capi import CProj

    p = Proj(Schema("uu", "u"), [key(0), lval(0) - 3, -rval(1)], where=[rval(1).ge(lval(1)), lval(0).lt(-2).signed()])
    assert not p.is_fn and isinstance(p._c, CProj)
    q = CProj()
    q.out_schema = Schema("uu", "u").c()
    q.n_pred = 2
    q.out[0] = Expr(capi.OP_COPY, key(0)).c()
    q.out[1] = Expr(capi.OP_SUB, lval(0), const(3)).c()
    q.out[2] = Expr(capi.OP_NEG, rval(1)).c()
    q.pred[0] = Pred(capi.CMP_GE, rval(1), lval(1)).c()
    q.pred[1] = Pred(capi.CMP_LT, lval(0), const(-2), True).c()
    assert bytes(p._c) == bytes(q)
    five = [col(0).eq(i) for i in range(5)]
    assert Proj(Schema("u"), [col(0)], five[:4]).is_fn is False and Proj(Schema("u"), [col(0)], five).is_fn is True
