"""Host-side handles: Schema, row expressions, Batch, Spine, and the backend.

A *backend* is a `CApi` plus one context; the product backend is
`runtime.Runtime` (CUDA library, fails loudly if it cannot load).  The
test-suite injects a second implementation of the same C ABI (the CPU
oracle, prefix ``orc_``) through `Backend` to check host logic without a
GPU — product code never constructs it.

Mirrors, on the host, the reference's `OrdZSet` / `OrdIndexedZSet` values
(crates/dbsp/src/trace/ord/zset_batch.rs:28-31, indexed_zset_batch.rs:27-41)
and the `zset!` / `indexed_zset!` literals (algebra/zset/zset_macro.rs:7-44).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Iterable, Sequence

import numpy as np

from . import _capi as capi
from ._capi import CApi, CExpr, CFold, CPred, CProj, CRowFn, CSchema, CSrc, as_u64, col_ptrs


@dataclass(frozen=True)
class Schema:
    """Row type: key lanes then value lanes, each 'u' (u64) or 'i' (i64)."""

    key: str
    val: str = ""

    @property
    def nk(self):
        return len(self.key)

    @property
    def nv(self):
        return len(self.val)

    @property
    def nl(self):
        return len(self.key) + len(self.val)

    @property
    def lanes(self):
        return self.key + self.val

    def c(self) -> CSchema:
        s = CSchema()
        s.n_key_lanes, s.n_val_lanes = self.nk, self.nv
        for i, t in enumerate(self.lanes):
            s.lane_types[i] = capi.I64 if t == "i" else capi.U64
        return s

    @staticmethod
    def from_c(s: CSchema) -> "Schema":
        t = "".join("i" if s.lane_types[i] == capi.I64 else "u" for i in range(s.n_key_lanes + s.n_val_lanes))
        return Schema(t[: s.n_key_lanes], t[s.n_key_lanes :])

    def reindex(self, nk: int) -> "Schema":
        return Schema(self.lanes[:nk], self.lanes[nk:])


def upsert_command_schema(table: Schema) -> Schema:
    """The command batch of a set / map input: the table's key lanes, then a u64 command lane and its value lanes."""
    return Schema(table.key, "u" + table.val)


# ---- declarative row expressions (stand in for the Rust closures) --------
# A closure whose lanes are single operations over two sources and whose filter is at most MAX_PREDS comparisons of
# two sources compiles to a `dbsp_proj`.  Anything else (nested arithmetic, %, abs, min/max, bitwise ops, shifts,
# where_, comparisons used as values, predicates combined with & | ~) compiles to a `dbsp_rowfn` program.
class Val:
    """Operator sugar of every row value.  Nesting builds a tree (Fn); Src overrides the operators that still fit
    one dbsp_expr."""

    is_bool = False   # the value is 0 or 1 (a comparison or a logical combination of comparisons)

    def __add__(self, o):
        return Fn(capi.FN_ADD, self, o)

    def __radd__(self, o):
        return Fn(capi.FN_ADD, o, self)

    def __sub__(self, o):
        return Fn(capi.FN_SUB, self, o)

    def __rsub__(self, o):
        return Fn(capi.FN_SUB, o, self)

    def __mul__(self, o):
        return Fn(capi.FN_MUL, self, o)

    def __rmul__(self, o):
        return Fn(capi.FN_MUL, o, self)

    def __floordiv__(self, o):
        """signed, truncating (Rust `/` on i64), x // 0 = 0"""
        return Fn(capi.FN_DIV, self, o)

    def __mod__(self, o):
        """signed remainder with the sign of the dividend (Rust `%` on i64), x % 0 = 0"""
        return Fn(capi.FN_REM, self, o)

    def divu(self, o):
        return Fn(capi.FN_DIVU, self, o)

    def remu(self, o):
        return Fn(capi.FN_REMU, self, o)

    def __neg__(self):
        return Fn(capi.FN_NEG, self)

    def __abs__(self):
        return Fn(capi.FN_ABS, self)

    def min(self, o):
        """unsigned unless .signed()"""
        return Fn(capi.FN_MINU, self, o)

    def max(self, o):
        return Fn(capi.FN_MAXU, self, o)

    def __and__(self, o):
        return Fn(capi.FN_AND, self, o)

    def __rand__(self, o):
        return Fn(capi.FN_AND, o, self)

    def __or__(self, o):
        return Fn(capi.FN_OR, self, o)

    def __ror__(self, o):
        return Fn(capi.FN_OR, o, self)

    def __xor__(self, o):
        return Fn(capi.FN_XOR, self, o)

    def __rxor__(self, o):
        return Fn(capi.FN_XOR, o, self)

    def __invert__(self):
        """logical NOT of a condition, bitwise NOT of any other value"""
        return Fn(capi.FN_LNOT if self.is_bool else capi.FN_BNOT, self)

    def __lshift__(self, o):
        return Fn(capi.FN_SHL, self, o)

    def __rshift__(self, o):
        """logical shift; .signed() makes it arithmetic"""
        return Fn(capi.FN_SHR, self, o)

    # comparison sugar -> Pred (unsigned unless .signed()), usable as a filter and as a 0 / 1 value
    def _cmp(self, op, o):
        return Pred(op, self, _val(o))

    def eq(self, o):
        return self._cmp(capi.CMP_EQ, o)

    def ne(self, o):
        return self._cmp(capi.CMP_NE, o)

    def lt(self, o):
        return self._cmp(capi.CMP_LT, o)

    def le(self, o):
        return self._cmp(capi.CMP_LE, o)

    def gt(self, o):
        return self._cmp(capi.CMP_GT, o)

    def ge(self, o):
        return self._cmp(capi.CMP_GE, o)

    def isin(self, codes):
        """membership in a set of small codes (< 64)"""
        mask = 0
        for c in codes:
            assert 0 <= c < 64
            mask |= 1 << c
        if mask >= 1 << 63:
            mask -= 1 << 64
        return self._cmp(capi.CMP_IN, mask)


class Src(Val):
    def __init__(self, kind, idx=0, cst=0):
        self.kind, self.idx, self.cst = kind, idx, cst

    def c(self) -> CSrc:
        s = CSrc()
        s.kind, s.idx, s.cst = self.kind, self.idx, self.cst
        return s

    def emit(self, code):
        code.append((capi.FN_PUSH, self.kind, self.idx, self.cst))

    # arithmetic of two sources -> Expr (one dbsp_expr); with a tree operand -> Fn
    def _op(self, op, o, tree_op):
        if isinstance(o, Val) and not isinstance(o, Src):
            return Fn(tree_op, self, o)
        return Expr(op, self, _src(o))

    def __neg__(self):
        return Expr(capi.OP_NEG, self)

    def __add__(self, o):
        return self._op(capi.OP_ADD, o, capi.FN_ADD)

    def __sub__(self, o):
        return self._op(capi.OP_SUB, o, capi.FN_SUB)

    def __mul__(self, o):
        return self._op(capi.OP_MUL, o, capi.FN_MUL)

    def __floordiv__(self, o):
        return self._op(capi.OP_DIV, o, capi.FN_DIV)


def _src(x):
    return x if isinstance(x, Src) else Src(capi.SRC_CONST, 0, int(x))


def _val(x):
    return x if isinstance(x, Val) else Src(capi.SRC_CONST, 0, int(x))


def key(i):
    return Src(capi.SRC_KEY, i)


def lval(i):
    return Src(capi.SRC_LVAL, i)


def rval(i):
    return Src(capi.SRC_RVAL, i)


val = lval  # single-input operators (map_index / weigh): the batch's value lanes
col = lval  # raw event tables: column index


def const(c):
    return Src(capi.SRC_CONST, 0, int(c))


def fanout_index():
    """j, the index (0 .. fanout-1) of the output a fan-out closure is generating (`Proj(..., fanout=n)`)"""
    return Src(capi.SRC_FANOUT)


def acc(i):
    """word i of a Fold's accumulator (its step and output programs only)"""
    return Src(capi.SRC_ACC, i)


def weight():
    """the weight of the value a Fold's step is applied to (summed over the trace's batches), as i64 bits"""
    return Src(capi.SRC_WEIGHT)


def where_(c, a, b):
    """`if c { a } else { b }` (c non-zero = true)"""
    return Fn(capi.FN_SELECT, c, a, b)


_EXPR_FN = {capi.OP_NEG: capi.FN_NEG, capi.OP_ADD: capi.FN_ADD, capi.OP_SUB: capi.FN_SUB, capi.OP_MUL: capi.FN_MUL,
            capi.OP_DIV: capi.FN_DIV}


class Expr(Val):
    def __init__(self, op, a, b=None):
        self.op, self.a, self.b = op, a, b if b is not None else Src(capi.SRC_CONST)

    def c(self) -> CExpr:
        e = CExpr()
        e.op, e.a, e.b = self.op, self.a.c(), self.b.c()
        return e

    def emit(self, code):
        self.a.emit(code)
        if self.op >= capi.OP_ADD:
            self.b.emit(code)
        if self.op != capi.OP_COPY:
            code.append((_EXPR_FN[self.op], 0, 0, 0))


def _expr(x) -> Expr:
    if isinstance(x, Expr):
        return x
    return Expr(capi.OP_COPY, _src(x))


def _lane(x):
    """an output lane: an Expr when it fits one dbsp_expr, else the tree"""
    if isinstance(x, Expr) or not isinstance(x, Val) or isinstance(x, Src):
        return _expr(x)
    return x


_CMP_FN = {capi.CMP_EQ: (capi.FN_EQ, capi.FN_EQ), capi.CMP_NE: (capi.FN_NE, capi.FN_NE),
           capi.CMP_LT: (capi.FN_LTU, capi.FN_LT), capi.CMP_LE: (capi.FN_LEU, capi.FN_LE),
           capi.CMP_GT: (capi.FN_GTU, capi.FN_GT), capi.CMP_GE: (capi.FN_GEU, capi.FN_GE),
           capi.CMP_IN: (capi.FN_IN, capi.FN_IN)}


class Pred(Val):
    is_bool = True

    def __init__(self, cmp, a, b, is_signed=False):
        self.cmp, self.a, self.b, self.is_signed = cmp, a, b, is_signed

    def signed(self):
        return Pred(self.cmp, self.a, self.b, True)

    def fits(self):
        return isinstance(self.a, Src) and isinstance(self.b, Src)

    def c(self) -> CPred:
        p = CPred()
        p.cmp, p.is_signed, p.a, p.b = self.cmp, int(self.is_signed), self.a.c(), self.b.c()
        return p

    def emit(self, code):
        self.a.emit(code)
        self.b.emit(code)
        code.append((_CMP_FN[self.cmp][int(self.is_signed)], 0, 0, 0))


_BOOL_FN = {capi.FN_LNOT, capi.FN_EQ, capi.FN_NE, capi.FN_LT, capi.FN_LE, capi.FN_GT, capi.FN_GE, capi.FN_LTU,
            capi.FN_LEU, capi.FN_GTU, capi.FN_GEU, capi.FN_IN}
_SIGNED_FN = {capi.FN_MINU: capi.FN_MIN, capi.FN_MAXU: capi.FN_MAX, capi.FN_SHR: capi.FN_SAR}


class Fn(Val):
    """An expression tree node: a row-function instruction over its operand trees."""

    def __init__(self, op, *args):
        self.op, self.args = op, [_val(a) for a in args]
        self.is_bool = op in _BOOL_FN or (op in (capi.FN_AND, capi.FN_OR) and all(a.is_bool for a in self.args)) or (
            op == capi.FN_SELECT and self.args[1].is_bool and self.args[2].is_bool)

    def signed(self):
        """min / max / >> in their signed forms"""
        assert self.op in _SIGNED_FN, "only min, max and >> have a signed form"
        return Fn(_SIGNED_FN[self.op], *self.args)

    def emit(self, code):
        for a in self.args:
            a.emit(code)
        code.append((self.op, 0, 0, 0))


def _i64(c):
    c = int(c) & ((1 << 64) - 1)
    return c - (1 << 64) if c >= 1 << 63 else c


def compile_rowfn(schema: Schema, out: Sequence, where: Sequence = ()) -> CRowFn:
    """The postfix program of a closure: the output lanes in order, then the keep flag (the AND of `where`)."""
    code = _compile_code(out, where)
    f = CRowFn()
    f.out_schema = schema.c()
    f.n_insn = len(code)
    for i, (op, kind, idx, cst) in enumerate(code):
        f.code[i].op, f.code[i].kind, f.code[i].idx, f.code[i].cst = op, kind, idx, _i64(cst)
    return f


def compile_fold_step(step: Sequence, where: Sequence = ()) -> list:
    """A Fold's step program: its n_acc (1 .. MAX_ACC) new accumulator words in order, then the keep flag (the AND of
    `where`).  The words are untyped, so no schema bounds them; the stack holds n_acc + 1 <= MAX_STACK values."""
    if not 1 <= len(step) <= capi.MAX_ACC:
        raise ValueError(f"Fold: the step gives {len(step)} accumulator words; an accumulator has 1..{capi.MAX_ACC}")
    return _compile_code(step, where)


def _compile_code(out: Sequence, where: Sequence) -> list:
    code = []
    for o in out:
        _val(o).emit(code)
    conds = [_val(w) for w in where]
    if not conds:
        code.append((capi.FN_PUSH, capi.SRC_CONST, 0, 1))
    for i, w in enumerate(conds):
        w.emit(code)
        if not w.is_bool:
            code += [(capi.FN_PUSH, capi.SRC_CONST, 0, 0), (capi.FN_NE, 0, 0, 0)]
        if i:
            code.append((capi.FN_AND, 0, 0, 0))
    if len(code) > capi.MAX_INSNS:
        raise ValueError(f"the closure needs {len(code)} instructions; a row function has at most {capi.MAX_INSNS}")
    return code


def compile_fold(init: Sequence[int], step_code: list, output: CRowFn) -> CFold:
    f = CFold()
    f.n_acc, f.n_step = len(init), len(step_code)
    for i, x in enumerate(init):
        f.init[i] = int(x) & ((1 << 64) - 1)
    for i, (op, kind, idx, cst) in enumerate(step_code):
        f.step[i].op, f.step[i].kind, f.step[i].idx, f.step[i].cst = op, kind, idx, _i64(cst)
    f.output = output
    return f


def _reads_fanout(x) -> bool:
    if isinstance(x, Src):
        return x.kind == capi.SRC_FANOUT
    if isinstance(x, (Expr, Pred)):
        return _reads_fanout(x.a) or _reads_fanout(x.b)
    if isinstance(x, Fn):
        return any(_reads_fanout(a) for a in x.args)
    return False


class Proj:
    """join_func / flat_map closure: output lanes + filter.  A `dbsp_proj` when it fits one (lanes of one operation
    over two sources, at most MAX_PREDS comparisons of two sources, AND-ed), else a `dbsp_rowfn` (is_fn).

    `fanout=n` makes it a flat_map closure that returns an iterator (filter_map.rs:124-160): the closure runs n times
    per input row with fanout_index() = 0 .. n-1, and each run whose filter holds yields one row (is_fanout, the
    `_fanout` entry points).  A closure with fanout 1 that never reads fanout_index() is an ordinary one."""

    def __init__(self, schema: Schema, out: Sequence, where: Sequence = (), fanout: int = 1):
        assert len(out) == schema.nl, "one expression per output lane"
        self.schema, self.out, self.where = schema, [_lane(o) for o in out], list(where)
        self.fanout = int(fanout)
        self.is_fanout = self.fanout != 1 or any(_reads_fanout(x) for x in self.out + self.where)
        self.is_fn = self.is_fanout or not (all(isinstance(e, Expr) for e in self.out) and len(self.where) <= capi.MAX_PREDS
                                            and all(isinstance(w, Pred) and w.fits() for w in self.where))
        if self.is_fn:
            self._c = compile_rowfn(schema, self.out, self.where)
            return
        p = CProj()
        p.out_schema = schema.c()
        p.n_pred = len(self.where)
        for i, e in enumerate(self.out):
            p.out[i] = e.c()
        for i, w in enumerate(self.where):
            p.pred[i] = w.c()
        self._c = p

    def c(self):
        return C.byref(self._c)

    def as_rowfn(self) -> "Proj":
        """The same closure compiled to a row function, whether or not it fits a dbsp_proj."""
        p = Proj.__new__(Proj)
        p.schema, p.out, p.where, p.is_fn = self.schema, self.out, self.where, True
        p.fanout, p.is_fanout = self.fanout, self.is_fanout
        p._c = compile_rowfn(self.schema, self.out, self.where)
        return p


def _factor(f):
    """weigh's f(k,v): a value (a dbsp_expr when it fits one) or a one-lane Proj, whose filter drops rows"""
    if isinstance(f, Proj):
        assert f.schema.nl == 1, "a weigh factor has one lane"
        if f.is_fanout:
            raise ValueError("weigh: a fan-out closure yields several rows; a weigh factor is one value per row")
        return "weigh_fn", f.as_rowfn()._c if not f.is_fn else f._c
    e = _lane(f)
    if isinstance(e, Expr):
        return "weigh", e.c()
    return "weigh_fn", compile_rowfn(Schema("u"), [e])


class Before:
    """RelOffset::Before(n) (time_series/range.rs): n time units before a timestamp."""
    after = False

    def __init__(self, n: int):
        if int(n) < 0:
            raise ValueError(f"{type(self).__name__}({n}): an offset is a non-negative magnitude")
        self.n = int(n)

    def __neg__(self):
        return (After if not self.after else Before)(self.n)

    def __eq__(self, o):
        return type(o) is type(self) and o.n == self.n

    def __repr__(self):
        return f"{type(self).__name__}({self.n})"

    def add(self, o, signed: bool):
        """RelOffset + RelOffset (range.rs), saturating in TS's type"""
        top = (1 << 63) - 1 if signed else (1 << 64) - 1
        if self.after == o.after:
            return type(self)(min(self.n + o.n, top))
        pos, neg = (self, o) if self.after else (o, self)   # After(pos.n) + Before(neg.n)
        return After(pos.n - neg.n) if pos.n >= neg.n else Before(neg.n - pos.n)

    def sub(self, o, signed: bool):
        return self.add(-o, signed)


class After(Before):
    """RelOffset::After(n) (time_series/range.rs): n time units after a timestamp."""
    after = True


def _ts_bounds(signed: bool):
    return (-(1 << 63), (1 << 63) - 1) if signed else (0, (1 << 64) - 1)


class RelRange:
    """RelRange{from, to} (time_series/range.rs) of a rolling aggregate: the range of a timestamp ts is
    [from(ts), to(ts)], each end Before(n) or After(n).  `frm` is not after `to`."""

    def __init__(self, frm: Before, to: Before):
        self.frm, self.to = frm, to

    def __repr__(self):
        return f"RelRange({self.frm!r}, {self.to!r})"

    def c(self) -> capi.CRelRange:
        r = capi.CRelRange()
        r.from_after, r.to_after, r.from_off, r.to_off = int(self.frm.after), int(self.to.after), self.frm.n, self.to.n
        return r

    def range_of(self, ts: int, signed: bool):
        """(from, to) of timestamp ts, or None when the range lies outside TS's type (range_of: a `from` After is a
        checked add, a `to` Before a checked subtract, the other ends saturate)"""
        lo, hi = _ts_bounds(signed)
        f = ts + self.frm.n if self.frm.after else ts - self.frm.n
        t = ts + self.to.n if self.to.after else ts - self.to.n
        if (self.frm.after and f > hi) or (not self.to.after and t < lo):
            return None
        return max(lo, min(hi, f)), max(lo, min(hi, t))

    def affected_range_of(self, ts: int, signed: bool):
        """(from, to) of the timestamps whose range holds ts, or None (affected_range_of)"""
        lo, hi = _ts_bounds(signed)
        f = ts - self.to.n if self.to.after else ts + self.to.n
        t = ts - self.frm.n if self.frm.after else ts + self.frm.n
        if (not self.to.after and f > hi) or (self.frm.after and t < lo):
            return None
        return max(lo, min(hi, f)), max(lo, min(hi, t))


class Batch:
    """Owning handle of an immutable device (or oracle) batch."""

    def __init__(self, be: "Backend", handle: int, schema: Schema | None = None):
        self.be, self.h = be, handle
        if schema is None:
            cs = CSchema()
            be.api.call("batch_schema", handle, C.byref(cs))
            schema = Schema.from_c(cs)
        self.schema = schema

    def __del__(self):
        try:
            if self.h:
                self.be.api._batch_free(self.h)
                self.h = None
        except Exception:
            pass

    def __len__(self):
        n = C.c_uint64()
        self.be.api.call("batch_len", self.h, C.byref(n))
        return n.value

    def key_count(self):
        n = C.c_uint64()
        self.be.api.call("batch_key_count", self.be.ctx, self.h, C.byref(n))
        return n.value

    def download(self):
        """Canonical vectors: dict(keys=[..], offs=.., vals=[..], diffs=..)."""
        s = self.schema
        n, nkeys = len(self), self.key_count()
        keys = [np.zeros(nkeys, np.uint64) for _ in range(s.nk)]
        vals = [np.zeros(n, np.uint64) for _ in range(s.nv)]
        offs = np.zeros(nkeys + 1, np.uint64) if s.nv else None
        diffs = np.zeros(n, np.int64)
        self.be.api.call(
            "batch_download_csr", self.be.ctx, self.h, col_ptrs(keys),
            offs.ctypes.data if offs is not None else None, col_ptrs(vals), diffs.ctypes.data,
        )
        for i, t in enumerate(s.key):
            if t == "i":
                keys[i] = keys[i].view(np.int64)
        for i, t in enumerate(s.val):
            if t == "i":
                vals[i] = vals[i].view(np.int64)
        return {"keys": keys, "offs": offs, "vals": vals, "diffs": diffs}

    def rows(self):
        """Flat list of (lane.., weight) python tuples (small batches)."""
        d = self.download()
        s = self.schema
        out = []
        if s.nv == 0:
            for i in range(len(d["diffs"])):
                out.append(tuple(int(k[i]) for k in d["keys"]) + (int(d["diffs"][i]),))
            return out
        nkeys = len(d["offs"]) - 1
        for k in range(nkeys):
            for v in range(int(d["offs"][k]), int(d["offs"][k + 1])):
                out.append(tuple(int(c[k]) for c in d["keys"]) + tuple(int(c[v]) for c in d["vals"]) + (int(d["diffs"][v]),))
        return out

    def last_key(self):
        k = (C.c_uint64 * capi.MAX_LANES)()
        valid = C.c_int32()
        self.be.api.call("batch_last_key", self.be.ctx, self.h, k, C.byref(valid))
        if not valid.value:
            return None
        out = []
        for i, t in enumerate(self.schema.key):
            v = int(k[i])
            out.append(v - (1 << 64) if (t == "i" and v >= 1 << 63) else v)
        return tuple(out)

    def __eq__(self, other):
        if not isinstance(other, Batch) or self.schema != other.schema:
            return False
        a, b = self.download(), other.download()
        eq = all(np.array_equal(x, y) for x, y in zip(a["keys"], b["keys"]))
        eq = eq and all(np.array_equal(x, y) for x, y in zip(a["vals"], b["vals"]))
        eq = eq and np.array_equal(a["diffs"], b["diffs"])
        if a["offs"] is not None:
            eq = eq and np.array_equal(a["offs"], b["offs"])
        return bool(eq)

    def __repr__(self):
        n = len(self)
        body = self.rows() if n <= 32 else f"{n} tuples"
        return f"Batch<{self.schema.key}|{self.schema.val}>({body})"


class Upload:
    """In-flight H2D copy of a raw table (keeps the host arrays alive)."""

    def __init__(self, be, handle, cols, weights):
        self.be, self.h, self._cols, self._w = be, handle, cols, weights

    def __del__(self):
        try:
            if self.h:
                self.be.api._upload_free(self.h)
                self.h = None
        except Exception:
            pass


class Download:
    """In-flight D2H copy of a batch's flat rows (keeps the destination arrays alive)."""

    def __init__(self, be, handle, n, cols, diffs):
        self.be, self.h, self.n, self.cols, self.diffs = be, handle, n, cols, diffs

    def finish(self):
        """Wait for the copy; returns (cols trimmed to n rows, diffs trimmed)."""
        if self.h:
            h, self.h = self.h, None
            self.be.api.call("download_finish", h)
        return [None if c is None else c[: self.n] for c in self.cols], None if self.diffs is None else self.diffs[: self.n]

    def __del__(self):
        try:
            if self.h:
                self.be.api._download_finish(self.h)
                self.h = None
        except Exception:
            pass


class Spine:
    """Owning handle of a trace (trace/spine_fueled.rs:107-119)."""

    def __init__(self, be: "Backend", schema: Schema, _handle=None):
        self.be, self.schema = be, schema
        if _handle is not None:
            self.h = _handle
            return
        h = C.c_void_p()
        be.api.call("spine_new", be.ctx, C.byref(schema.c()), C.byref(h))
        self.h = h.value

    def save(self, path: str):
        """Checkpoint the trace to `path` (dbsp_spine_save)."""
        self.be.api.call("spine_save", self.be.ctx, self.h, str(path).encode())

    @staticmethod
    def load(be: "Backend", path: str, schema: Schema) -> "Spine":
        """Resume a trace from a checkpoint written by save() — by this library or by the oracle."""
        h = C.c_void_p()
        be.api.call("spine_load", be.ctx, str(path).encode(), C.byref(h))
        return Spine(be, schema, _handle=h.value)

    def __del__(self):
        try:
            if self.h:
                self.be.api._spine_free(self.h)
                self.h = None
        except Exception:
            pass

    def insert(self, b: Batch):
        self.be.api.call("spine_insert", self.be.ctx, self.h, b.h)

    def consolidate(self) -> Batch:
        out = C.c_void_p()
        self.be.api.call("spine_consolidate", self.be.ctx, self.h, C.byref(out))
        return Batch(self.be, out.value, self.schema)

    def truncate_keys_below(self, key: Sequence[int]):
        k = (C.c_uint64 * capi.MAX_LANES)(*[int(x) & ((1 << 64) - 1) for x in key])
        self.be.api.call("spine_truncate_keys_below", self.be.ctx, self.h, k)

    def truncate_values_below(self, val: Sequence[int]):
        """Trace::truncate_values_below (spine_fueled.rs:644-656)."""
        v = (C.c_uint64 * capi.MAX_LANES)(*[int(x) & ((1 << 64) - 1) for x in val])
        self.be.api.call("spine_truncate_values_below", self.be.ctx, self.h, v)

    def exert(self, effort: int) -> int:
        """Trace::exert (spine_fueled.rs:627-634); returns the effort left."""
        e = C.c_int64(int(effort))
        self.be.api.call("spine_exert", self.be.ctx, self.h, C.byref(e))
        return e.value

    def stats(self):
        n, nb = C.c_uint64(), C.c_uint32()
        self.be.api.call("spine_len", self.h, C.byref(n), C.byref(nb))
        return n.value, nb.value


class Merger:
    """The fuelled Merger (trace/mod.rs:371-396): new_merger / work / done."""

    def __init__(self, be: "Backend", a: Batch, b: Batch, val_lower_bound: Sequence[int] | None = None):
        self.be, self.schema = be, a.schema
        self._keep = (a, b)
        h = C.c_void_p()
        be.api.call("merger_new", be.ctx, a.h, b.h, _lanes(val_lower_bound), C.byref(h))
        self.h = h.value

    def work(self, fuel: int) -> int:
        """Spend up to `fuel`; the returned fuel is > 0 iff the merge is complete."""
        f = C.c_int64(int(fuel))
        self.be.api.call("merger_work", self.be.ctx, self.h, C.byref(f))
        return f.value

    def done(self) -> Batch:
        out = C.c_void_p()
        h, self.h = self.h, None   # freed by the library on success
        try:
            self.be.api.call("merger_done", self.be.ctx, h, C.byref(out))
        except Exception:
            self.h = h
            raise
        return Batch(self.be, out.value, self.schema)

    def __del__(self):
        try:
            if self.h:
                self.be.api._merger_free(self.h)
                self.h = None
        except Exception:
            pass


class Batcher:
    """Batcher (trace/mod.rs:316-335) = MergeBatcher (merge_batcher/mod.rs:22-81)."""

    def __init__(self, be: "Backend", schema: Schema):
        self.be, self.schema = be, schema
        h = C.c_void_p()
        be.api.call("batcher_new", be.ctx, C.byref(schema.c()), C.byref(h))
        self.h = h.value

    def _push(self, fn, cols, weights):
        cols = [as_u64(c) for c in cols]
        n = len(cols[0]) if cols else 0
        w = np.ascontiguousarray(np.asarray(weights, dtype=np.int64)) if weights is not None else None
        self.be.api.call(fn, self.be.ctx, self.h, col_ptrs(cols), w.ctypes.data if w is not None else None, n, 0)

    def push_batch(self, cols: Sequence, weights=None):
        """Unsorted tuples, column-major host arrays (weights None = all +1)."""
        self._push("batcher_push", cols, weights)

    def push_rows(self, rows: Iterable[Sequence[int]]):
        rows = list(rows)
        if not rows:
            return
        arr = [[_wrap(r[l]) for r in rows] for l in range(self.schema.nl)]
        self.push_batch([np.array(a, dtype=np.uint64) for a in arr], [r[-1] for r in rows])

    def push_consolidated_batch(self, cols: Sequence, weights):
        """Rows already sorted, unique and non-zero."""
        self._push("batcher_push_consolidated", cols, weights)

    def tuples(self) -> int:
        n = C.c_uint64()
        self.be.api.call("batcher_tuples", self.h, C.byref(n))
        return n.value

    def seal(self) -> Batch:
        out = C.c_void_p()
        h, self.h = self.h, None   # consumed by the library
        self.be.api.call("batcher_seal", self.be.ctx, h, C.byref(out))
        return Batch(self.be, out.value, self.schema)

    def __del__(self):
        try:
            if self.h:
                self.be.api._batcher_free(self.h)
                self.h = None
        except Exception:
            pass


def _wrap(x):
    return int(x) & ((1 << 64) - 1)


_FANOUT_CALLS = {"batch_from_table", "batch_from_upload", "map_index"}


def _fn(call, proj: Proj):
    """the entry point for the closure's form: `call` for a dbsp_proj, `call_fn` for a dbsp_rowfn, `call_fanout`
    for a fan-out"""
    if getattr(proj, "is_fanout", False):
        if call not in _FANOUT_CALLS:
            raise ValueError(f"{call}: a fan-out closure applies to flat_map / flat_map_index and tables only")
        return call + "_fanout"
    return call + "_fn" if proj.is_fn else call


def _closure(proj: Proj):
    """the closure arguments of the entry point `_fn` picks: the struct, and a fan-out's n_out after it"""
    return (proj.c(), proj.fanout) if getattr(proj, "is_fanout", False) else (proj.c(),)


def _lanes(vals: Sequence[int] | None):
    if vals is None:
        return None
    return (C.c_uint64 * capi.MAX_LANES)(*[int(x) & ((1 << 64) - 1) for x in vals])


class Backend:
    """One C-ABI library + one context.  Operator-level calls, 1:1 with the
    header (see include/dbsp_b200.h for the reference file:line of each)."""

    name = "abstract"

    def __init__(self, api: CApi, device: int = 0):
        self.api = api
        ctx = C.c_void_p()
        api.call("ctx_create", device, C.byref(ctx))
        self.ctx = ctx.value
        self.device = device

    def close(self):
        if getattr(self, "ctx", None):
            self.api._ctx_destroy(self.ctx)
            self.ctx = None

    def sync(self):
        self.api.call("ctx_sync", self.ctx)

    def stats(self, reset=False):
        a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
        self.api.call("ctx_stats", self.ctx, C.byref(a), C.byref(b), C.byref(c), int(reset))
        n, us = C.c_uint64(), C.c_double()
        self.api.call("ctx_sync_stats", self.ctx, C.byref(n), C.byref(us), int(reset))
        return {"kernel_launches": a.value, "h2d_bytes": b.value, "d2h_bytes": c.value,
                "host_waits": n.value, "host_wait_ms": us.value / 1e3}

    def download_begin(self, batch: "Batch", cols: Sequence, diffs):
        """Queue the D2H copy of `batch`'s flat rows into caller-owned (pinned) arrays: cols[l] takes lane l,
        diffs the weights, each with room for len(batch) entries.  Returns a Download; .finish() waits."""
        cols = [None if c is None else as_u64(c) for c in cols]
        n = len(batch)
        for c in cols:
            assert c is None or len(c) >= n
        assert diffs is None or len(diffs) >= n
        ptrs = col_ptrs(cols)
        h = C.c_void_p()
        self.api.call("batch_download_begin", self.ctx, batch.h, ptrs, diffs.ctypes.data if diffs is not None else None,
                      C.byref(h))
        return Download(self, h.value, n, cols, diffs)

    def profile(self, enable=True):
        self.api.call("ctx_profile", self.ctx, int(enable))

    def profile_pause(self):
        """Stop recording per-kernel events; what was collected stays readable (a sampling window)."""
        self.api.call("ctx_profile", self.ctx, 2)

    def profile_read(self):
        """{kernel name: dict(launches, ms, alg_bytes)} since profile(True)."""
        out, i = {}, 0
        while True:
            name = C.create_string_buffer(32)
            n, ms, b = C.c_uint64(), C.c_double(), C.c_uint64()
            rc = self.api._ctx_profile_read(self.ctx, i, name, C.byref(n), C.byref(ms), C.byref(b))
            if rc != 0:
                break
            if n.value:
                out[name.value.decode()] = {"launches": n.value, "ms": ms.value, "alg_bytes": b.value}
            i += 1
        return out

    # -- construction ------------------------------------------------------
    def _out(self):
        return C.c_void_p()

    def batch_from_columns(self, schema: Schema, cols: Sequence, weights=None, n=None, on_device=False) -> Batch:
        """Batch::from_tuples over column-major inputs.  Host inputs are numpy
        arrays; device inputs are raw integer addresses (on_device=True)."""
        if not on_device:
            cols = [as_u64(c) for c in cols]
            n = len(cols[0]) if cols else (len(weights) if weights is not None else 0)
            if weights is not None:
                weights = np.ascontiguousarray(np.asarray(weights, dtype=np.int64))
            wptr = weights.ctypes.data if weights is not None else None
        else:
            wptr = weights
        out = self._out()
        self.api.call("batch_from_tuples", self.ctx, C.byref(schema.c()), col_ptrs(cols), wptr, n, int(on_device), C.byref(out))
        return Batch(self, out.value, schema)

    def batch_from_rows(self, schema: Schema, rows: Iterable[Sequence[int]]) -> Batch:
        """rows: (lane.., weight) tuples — the `zset!` literal."""
        rows = list(rows)
        if not rows:
            return self.batch_empty(schema)
        arr = np.array([[int(x) & ((1 << 64) - 1) for x in r] for r in rows], dtype=np.uint64)
        cols = [np.ascontiguousarray(arr[:, i]) for i in range(schema.nl)]
        w = np.ascontiguousarray(arr[:, schema.nl]).view(np.int64)
        return self.batch_from_columns(schema, cols, w)

    def batch_from_table(self, cols: Sequence, proj: Proj, weights=None, n=None, on_device=False) -> Batch:
        if not on_device:
            cols = [as_u64(c) for c in cols]
            n = len(cols[0])
            if weights is not None:
                weights = np.ascontiguousarray(np.asarray(weights, dtype=np.int64))
            wptr = weights.ctypes.data if weights is not None else None
        else:
            wptr = weights
        out = self._out()
        self.api.call(_fn("batch_from_table", proj), self.ctx, col_ptrs(cols), len(cols), wptr, n, int(on_device),
                      *_closure(proj), C.byref(out))
        return Batch(self, out.value, proj.schema)

    def upload_begin(self, cols: Sequence, col_mask: int = 0xFF, weights=None):
        """Start the H2D copy of a future step's table (pinned host columns)."""
        cols = [as_u64(c) for c in cols]
        n = len(cols[0])
        if weights is not None:
            weights = np.ascontiguousarray(np.asarray(weights, dtype=np.int64))
        up = C.c_void_p()
        self.api.call("upload_begin", self.ctx, col_ptrs(cols), len(cols), col_mask,
                      weights.ctypes.data if weights is not None else None, n, C.byref(up))
        return Upload(self, up.value, cols, weights)

    def batch_from_upload(self, up: "Upload", proj: Proj) -> Batch:
        out = self._out()
        self.api.call(_fn("batch_from_upload", proj), self.ctx, up.h, *_closure(proj), C.byref(out))
        return Batch(self, out.value, proj.schema)

    def proj_table_mask(self, proj: Proj) -> int:
        if getattr(proj, "is_fanout", False):
            return int(self.api._fanout_table_mask(proj.c()))
        return int((self.api._rowfn_table_mask if proj.is_fn else self.api._proj_table_mask)(proj.c()))

    def batch_from_sorted(self, schema: Schema, cols: Sequence, weights, n: int, on_device: bool) -> Batch:
        out = self._out()
        if not on_device:
            cols = [as_u64(c) for c in cols]
            weights = np.ascontiguousarray(np.asarray(weights, dtype=np.int64))
            wptr = weights.ctypes.data
        else:
            wptr = weights
        self.api.call("batch_from_sorted", self.ctx, C.byref(schema.c()), col_ptrs(cols), wptr, n, int(on_device), C.byref(out))
        return Batch(self, out.value, schema)

    def batch_empty(self, schema: Schema) -> Batch:
        out = self._out()
        self.api.call("batch_empty", self.ctx, C.byref(schema.c()), C.byref(out))
        return Batch(self, out.value, schema)

    # -- batch algebra -----------------------------------------------------
    def merge(self, a: Batch, b: Batch, val_lower_bound: Sequence[int] | None = None) -> Batch:
        out = self._out()
        if val_lower_bound is None:
            self.api.call("batch_merge", self.ctx, a.h, b.h, C.byref(out))
        else:
            self.api.call("batch_merge_bounded", self.ctx, a.h, b.h, _lanes(val_lower_bound), C.byref(out))
        return Batch(self, out.value, a.schema)

    def batcher(self, schema: Schema) -> "Batcher":
        return Batcher(self, schema)

    def merger(self, a: Batch, b: Batch, val_lower_bound: Sequence[int] | None = None) -> "Merger":
        return Merger(self, a, b, val_lower_bound)

    def truncate_keys_below(self, b: Batch, key: Sequence[int]) -> Batch:
        out = self._out()
        self.api.call("batch_truncate_keys_below", self.ctx, b.h, _lanes(key), C.byref(out))
        return Batch(self, out.value, b.schema)

    def neg(self, a: Batch) -> Batch:
        out = self._out()
        self.api.call("batch_neg", self.ctx, a.h, C.byref(out))
        return Batch(self, out.value, a.schema)

    def reindex(self, a: Batch, nk: int) -> Batch:
        out = self._out()
        self.api.call("batch_reindex", self.ctx, a.h, nk, C.byref(out))
        return Batch(self, out.value, a.schema.reindex(nk))

    # -- operators ---------------------------------------------------------
    def join_delta_trace(self, delta: Batch, trace: Spine, proj: Proj, delta_is_left=True) -> Batch:
        out = self._out()
        self.api.call(_fn("join_delta_trace", proj), self.ctx, delta.h, trace.h, proj.c(), int(delta_is_left), C.byref(out))
        return Batch(self, out.value, proj.schema)

    def join_batches(self, left: Batch, right: Batch, proj: Proj) -> Batch:
        out = self._out()
        self.api.call(_fn("join_batches", proj), self.ctx, left.h, right.h, proj.c(), C.byref(out))
        return Batch(self, out.value, proj.schema)

    def semijoin(self, pairs: Batch, keys: Batch) -> Batch:
        out = self._out()
        self.api.call("semijoin", self.ctx, pairs.h, keys.h, C.byref(out))
        return Batch(self, out.value, Schema(pairs.schema.lanes))   # OrdZSet<(K, V)> (semijoin.rs:47)

    def aggregate_delta(self, delta: Batch, in_trace: Spine, out_trace: Spine, kind: int) -> Batch:
        out = self._out()
        self.api.call("aggregate_delta", self.ctx, delta.h, in_trace.h, out_trace.h, kind, C.byref(out))
        return Batch(self, out.value, out_trace.schema)

    def aggregate_fold(self, delta: Batch, in_trace: Spine, out_trace: Spine, fold) -> Batch:
        """aggregate_delta with a Fold (circuit.Fold, or anything with a CFold `_c`) as the aggregator."""
        out = self._out()
        self.api.call("aggregate_fold", self.ctx, delta.h, in_trace.h, out_trace.h, C.byref(fold._c), C.byref(out))
        return Batch(self, out.value, out_trace.schema)

    def upsert_commands(self, table: Schema, cols: Sequence, insert=None, n=None, seq0: int = 0, on_device=False) -> Batch:
        """The commands of a set / map input as a batch (dbsp_upsert_commands): command i is row i of `cols` (the
        table's lanes) with the sequence number seq0 + i; `insert` (one flag per command, None: all insert) tells
        inserts from deletes.  Host inputs are numpy arrays; device inputs are raw addresses (on_device=True)."""
        if not on_device:
            cols = [as_u64(c) for c in cols]
            n = len(cols[0]) if cols else 0
            if insert is not None:
                insert = np.ascontiguousarray(np.asarray(insert) != 0, dtype=np.uint8)
            iptr = insert.ctypes.data if insert is not None else None
        else:
            iptr = insert
        out = self._out()
        self.api.call("upsert_commands", self.ctx, C.byref(table.c()), col_ptrs(cols), iptr, n, seq0, int(on_device),
                      C.byref(out))
        return Batch(self, out.value, upsert_command_schema(table))

    def upsert_delta(self, cmds: Batch, table: Spine) -> Batch:
        """Upsert::eval of a command batch against the table's trace: the table's change (dbsp_upsert_delta)."""
        out = self._out()
        self.api.call("upsert_delta", self.ctx, cmds.h, table.h, C.byref(out))
        return Batch(self, out.value, table.schema)

    def rolling_aggregate(self, delta: Batch, in_trace: Spine, out_trace: Spine, rng: RelRange, kind: int,
                          f: Proj | None = None) -> Batch:
        """PartitionedRollingAggregate::eval (dbsp_rolling_aggregate): the change of the rolling aggregate's output
        at the times `delta` affects.  `f` is LINEAR's row function (a Proj of value lanes only), None otherwise."""
        out = self._out()
        fc = None if f is None else C.byref(f._c if f.is_fn else f.as_rowfn()._c)
        self.api.call("rolling_aggregate", self.ctx, delta.h, in_trace.h, out_trace.h, C.byref(rng.c()), kind, fc,
                      C.byref(out))
        return Batch(self, out.value, out_trace.schema)

    def weigh(self, b: Batch, f, mode: int) -> Batch:
        """f: a value of the key / value lanes, or a one-lane Proj whose filter drops rows."""
        out = self._out()
        call, e = _factor(f)
        self.api.call(call, self.ctx, b.h, C.byref(e), mode, C.byref(out))
        return Batch(self, out.value)

    def distinct_delta(self, delta: Batch, integral: Spine) -> Batch:
        out = self._out()
        self.api.call("distinct_delta", self.ctx, delta.h, integral.h, C.byref(out))
        return Batch(self, out.value, delta.schema)

    def antijoin_delta(self, delta: Batch, trace: Spine, key_delta: Batch, key_trace: Spine) -> Batch:
        """delta·(1 − key_trace(k)) − trace ⋉ key_delta: the antijoin's change, with the keys' distinct-value counts
        (OrdZSet<K>) in place of distinct(other)."""
        out = self._out()
        self.api.call("antijoin_delta", self.ctx, delta.h, trace.h, key_delta.h, key_trace.h, C.byref(out))
        return Batch(self, out.value, delta.schema)

    def stream_distinct(self, b: Batch) -> Batch:
        out = self._out()
        self.api.call("stream_distinct", self.ctx, b.h, C.byref(out))
        return Batch(self, out.value, b.schema)

    def window_delta(self, trace: Spine, delta: Batch, prev, cur) -> Batch:
        def arr(k):
            return (C.c_uint64 * capi.MAX_LANES)(*[int(x) & ((1 << 64) - 1) for x in k])

        s0, e0 = (arr(prev[0]), arr(prev[1])) if prev is not None else (arr(cur[0]), arr(cur[1]))
        out = self._out()
        self.api.call("window_delta", self.ctx, trace.h, delta.h, int(prev is not None), s0, e0, arr(cur[0]), arr(cur[1]), C.byref(out))
        return Batch(self, out.value, delta.schema)

    def map_index(self, b: Batch, proj: Proj) -> Batch:
        out = self._out()
        self.api.call(_fn("map_index", proj), self.ctx, b.h, *_closure(proj), C.byref(out))
        return Batch(self, out.value, proj.schema)

    def shard_partition(self, b: Batch, n_shards: int):
        outs = (C.c_void_p * n_shards)()
        self.api.call("shard_partition", self.ctx, b.h, n_shards, outs)
        return [Batch(self, outs[i], b.schema) for i in range(n_shards)]

    # -- communication between replicas (include/dbsp_b200.h "communication") ------
    def comm_create(self, rank: int, world: int, slot_bytes: int = 0) -> bytes:
        blob = (C.c_uint8 * capi.COMM_BLOB_BYTES)()
        self.api.call("comm_create", self.ctx, rank, world, slot_bytes, blob)
        return bytes(blob)

    def comm_connect(self, blobs: bytes):
        buf = (C.c_uint8 * len(blobs)).from_buffer_copy(blobs)
        self.api.call("comm_connect", self.ctx, buf)

    def comm_destroy(self):
        if getattr(self, "ctx", None):
            self.api.call("comm_destroy", self.ctx)

    def comm_info(self):
        r, w, b = C.c_int32(), C.c_int32(), C.c_uint64()
        self.api.call("comm_info", self.ctx, C.byref(r), C.byref(w), C.byref(b))
        return r.value, w.value, b.value

    def shard(self, b: Batch) -> Batch:
        out = self._out()
        self.api.call("shard", self.ctx, b.h, C.byref(out))
        return Batch(self, out.value, b.schema)

    def shard2(self, a: Batch, b: Batch):
        oa, ob = self._out(), self._out()
        self.api.call("shard2", self.ctx, a.h, b.h, C.byref(oa), C.byref(ob))
        return Batch(self, oa.value, a.schema), Batch(self, ob.value, b.schema)

    def gather(self, b: Batch, root: int = 0) -> Batch:
        out = self._out()
        self.api.call("gather", self.ctx, b.h, root, C.byref(out))
        return Batch(self, out.value, b.schema)

    def allreduce_max(self, x: int) -> int:
        v = C.c_uint64(int(x) & ((1 << 64) - 1))
        self.api.call("allreduce_max_u64", self.ctx, C.byref(v))
        return v.value

    # -- flat column access for the exchange (overridden per backend) -------
    def batch_flat_tensors(self, b: Batch):
        """(list of per-lane torch tensors, weight tensor) of the flat rows."""
        raise NotImplementedError

    def batch_from_flat_tensors(self, schema: Schema, cols, weights) -> Batch:
        raise NotImplementedError
