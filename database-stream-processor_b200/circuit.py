"""Stream / operator API for the Z-set delta hot path.

Host-side mirror of the reference's `RootCircuit` + `Stream` operator surface
(crates/dbsp/src/circuit/circuit_builder.rs:1403-1433, operator/*.rs) for the
operators on the hot path.  A circuit is a static DAG built once; `step()`
evaluates every node once in creation (= dependency) order, exactly like the
reference's schedulers (circuit/schedule/static_scheduler.rs:52-87).  All
data work is done by the backend (the CUDA library behind include/dbsp_b200.h).

Rust closures become declarative `Proj` / expression objects (zset.py).
Stateful operators own their traces; the `z^-1` delays of the reference's
feedback loops are realised by the order of trace inserts inside `eval`.
"""
from __future__ import annotations

from typing import Callable, Sequence

import numpy as np

from . import _capi as capi
from .zset import (After, Backend, Batch, Before, Expr, Fn, Pred, Proj, RelRange, Schema, Spine, Src, acc, compile_fold,
                   compile_fold_step, const, key, lval, rval, upsert_command_schema)


class Max:  # operator/aggregate/max.rs:36-55
    kind = capi.AGG_MAX


class Min:  # operator/aggregate/min.rs:38-57
    kind = capi.AGG_MIN


class FoldCount:  # Fold counting distinct values (aggregate/mod.rs:908-916)
    kind = capi.AGG_FOLD_COUNT


class FoldSum:  # Fold summing distinct values (aggregate/mod.rs:918-929)
    kind = capi.AGG_FOLD_SUM


class Fold:
    """Fold::new / Fold::with_output (operator/aggregate/fold.rs), the general aggregator: per key, `init`, then
    `step` applied in value order to each value whose weight (summed over the trace) is non-zero, then `output`.

    init: the accumulator's n_acc (1..15) words.  step: n_acc expressions, the new words, over key(i), lval(i) / val(i)
    (the value's lanes), acc(i), weight() and constants.  where: the step's keep condition(s); a value for which it
    does not hold leaves the accumulator unchanged.  output: a Proj over key(i) / acc(i) with value lanes only (its
    filter drops the key's row); by default the accumulator itself, typed u (n_acc <= 8).  A key with no value of
    non-zero weight has no row.  Fold is not a semigroup (UnimplementedSemigroup): every key is walked serially."""

    def __init__(self, init: Sequence[int], step: Sequence, output: Proj | None = None, where=None):
        init = [int(x) for x in init]
        if len(step) != len(init):
            raise ValueError(f"Fold: init has {len(init)} accumulator words and step gives {len(step)}")
        where = [] if where is None else list(where) if isinstance(where, (list, tuple)) else [where]
        code = compile_fold_step(step, where)
        if output is None:
            if len(init) > capi.MAX_LANES:
                raise ValueError(f"Fold: an accumulator of {len(init)} words needs an output of at most {capi.MAX_LANES} lanes")
            output = Proj(Schema("", "u" * len(init)), [acc(i) for i in range(len(init))])
        if output.schema.nk != 0:
            raise ValueError("Fold: the output has key lanes; it gives the key's value lanes only")
        if output.is_fanout:
            raise ValueError("Fold: the output is a fan-out closure; a key has one output")
        self.init, self.step, self.where, self.output = init, list(step), where, output
        self._c = compile_fold(init, code, output._c if output.is_fn else output.as_rowfn()._c)


class Linear:
    """The linear rolling aggregator (rolling_aggregate.rs LinearAggregator): per output lane of `f`, the sum of
    f(pk, v) * weight over the window, wrapping in i64.  `f` is a Proj with value lanes only over key(i) (the partition
    key), lval(i) / val(i) (the lanes after the timestamp) and constants; a row its filter drops adds 0."""

    kind = capi.ROLLING_LINEAR

    def __init__(self, f: Proj):
        if f.schema.nk != 0 or f.schema.nv == 0:
            raise ValueError(f"Linear: f must have value lanes only, has schema {f.schema}")
        if f.is_fanout:
            raise ValueError("Linear: f is a fan-out closure; a row has one term")
        self.f = f


def _rolling_kind(aggregator):
    """(kind, f) of a rolling aggregator: Max, Min or Linear(f)"""
    if isinstance(aggregator, Linear):
        return capi.ROLLING_LINEAR, aggregator.f
    if aggregator is Max or isinstance(aggregator, Max):
        return capi.ROLLING_MAX, None
    if aggregator is Min or isinstance(aggregator, Min):
        return capi.ROLLING_MIN, None
    raise ValueError(f"partitioned_rolling_aggregate: {aggregator!r} is not Max, Min or Linear(f)")


class _KeyCounts:
    """N(k), the number of distinct (k, v) rows of a stream's integral, as a trace of OrdZSet<K> counts.  step()
    returns the change of the counts: distinct_delta's ±1 rows with their values dropped, which consolidation sums
    per key."""

    def __init__(self, be: Backend, schema: Schema):
        self.be = be
        self.keys = Proj(Schema(schema.key), [key(i) for i in range(schema.nk)])
        self.trace = Spine(be, Schema(schema.key))

    def step(self, delta: Batch, delayed_integral: Spine) -> Batch:
        dn = self.be.map_index(self.be.distinct_delta(delta, delayed_integral), self.keys)
        self.trace.insert(dn)
        return dn


def _zero_src(x, kind):
    """The expression tree `x` with every source of `kind` read as 0."""
    if isinstance(x, Src):
        return const(0) if x.kind == kind else x
    if isinstance(x, Expr):
        return Expr(x.op, _zero_src(x.a, kind), _zero_src(x.b, kind))
    if isinstance(x, Pred):
        return Pred(x.cmp, _zero_src(x.a, kind), _zero_src(x.b, kind), x.is_signed)
    return Fn(x.op, *[_zero_src(a, kind) for a in x.args])


class Node:
    def __init__(self, circuit: "RootCircuit", inputs: Sequence["Node"], fn: Callable, name: str):
        self.circuit, self.inputs, self.fn, self.name = circuit, list(inputs), fn, name
        self.value = None
        circuit.nodes.append(self)

    def eval(self):
        self.value = self.fn(*[i.value for i in self.inputs])


class InputHandle:
    """CollectionHandle (operator/input.rs:664-703): rows appended between
    steps form the next step's batch."""

    def __init__(self, circuit, schema: Schema):
        self.circuit, self.schema, self.pending = circuit, schema, []

    def append(self, rows):
        """rows: iterable of (lane.., weight)."""
        self.pending.extend(rows)

    def push(self, *row):
        """push(k.., w) (operator/input.rs:676-681): one (lane.., weight) update."""
        self.pending.append(tuple(row))

    def clear_input(self):
        """clear_input (operator/input.rs:697-703): drop the updates buffered since the last step."""
        self.pending = []

    def _take(self) -> Batch:
        rows, self.pending = self.pending, []
        return self.circuit.be.batch_from_rows(self.schema, rows)


class TableHandle:
    """Input of a raw column-major event table (no order, optional weights).
    `set(cols, weights=None)` with host numpy columns, or
    `set_device(ptrs, n)` with resident device columns."""

    def __init__(self):
        self.cur = None

    def set(self, cols, weights=None):
        self.cur = ("host", list(cols), weights, None)

    def set_device(self, ptrs, n, weights=None):
        self.cur = ("dev", list(ptrs), weights, int(n))

    def set_upload(self, upload):
        """upload: an `Upload` started with Backend.upload_begin for this step
        (pipelined ingest; its column mask must cover `TableStream.table_mask()`)."""
        self.cur = ("upload", upload, None, None)

    def _take(self):
        cur, self.cur = self.cur, None
        return cur


_M64 = (1 << 64) - 1


class UpsertHandle:
    """UpsertHandle (operator/input.rs:747-882): the commands of a set or map input table.  The commands buffered
    between steps form the next step's; per key only the last one counts.  A key is an int (one key lane) or a tuple
    of the key lanes, a map's value likewise for the value lanes.

    A set's command is push(key, insert) with a bool; a map's is push(key, value), value None deleting the key.
    For bulk loads, append_columns(cols, insert=None) takes host numpy columns and append_device(ptrs, n,
    insert=None) resident device columns: the table's lanes (a delete's value lanes are ignored) and one flag per
    command (None: every command inserts).  Appends keep their order within a step, whatever their kind."""

    # A step's commands on worker r are numbered from r << SEQ_RANK_SHIFT: a key's commands are ordered by worker
    # rank, then push order, and a worker may take up to 2^40 commands per step.
    SEQ_RANK_SHIFT = 40

    def __init__(self, circuit, schema: Schema, is_map: bool):
        self.circuit, self.schema, self.is_map = circuit, schema, is_map
        self.pending = []   # ("rows", [(lanes, insert)]) | ("host", cols, insert) | ("dev", ptrs, n, insert)

    @staticmethod
    def _lanes(x, n, what):
        t = tuple(x) if isinstance(x, (tuple, list)) else (x,)
        if len(t) != n or not all(isinstance(v, (int, np.integer)) and not isinstance(v, (bool, np.bool_)) for v in t):
            raise ValueError(f"UpsertHandle: {what} must be {n} integer lane(s), got {x!r}")
        return t

    def _command(self, key, value):
        s = self.schema
        k = self._lanes(key, s.nk, "a key")
        if not self.is_map:
            if not isinstance(value, (bool, np.bool_)):
                raise ValueError(f"UpsertHandle: a set's command is (key, bool), got the value {value!r}")
            return k, bool(value)
        if value is None:
            return k + (0,) * s.nv, False
        return k + self._lanes(value, s.nv, "a value"), True

    def _rows(self, rows):
        if not rows:
            return
        if not self.pending or self.pending[-1][0] != "rows":
            self.pending.append(("rows", []))
        self.pending[-1][1].extend(rows)

    def push(self, key, value):
        """push (input.rs:802-815): one command."""
        self._rows([self._command(key, value)])

    def append(self, commands):
        """append (input.rs:836-877): (key, value) commands in order; a malformed one raises before any is taken."""
        self._rows([self._command(k, v) for k, v in commands])

    def append_columns(self, cols, insert=None):
        """Commands as host columns: the table's lanes, and one insert flag per command (None: all insert)."""
        cols = [np.asarray(c) for c in cols]
        n = self._check_columns(len(cols), [len(c) for c in cols], insert)
        if n:
            self.pending.append(("host", cols, insert))

    def append_device(self, ptrs, n, insert=None):
        """Commands as resident device columns (raw addresses of n u64 each) and an optional device array of n u8
        insert flags."""
        ptrs = list(ptrs)
        self._check_columns(len(ptrs), [int(n)] * len(ptrs), None)
        if int(n):
            self.pending.append(("dev", ptrs, int(n), insert))

    def _check_columns(self, n_cols, lens, insert):
        s = self.schema
        if n_cols != s.nl:
            raise ValueError(f"UpsertHandle: the table has {s.nl} lanes, got {n_cols} columns")
        if len(set(lens)) > 1:
            raise ValueError(f"UpsertHandle: columns of different lengths {lens}")
        n = lens[0]
        if insert is not None and len(insert) != n:
            raise ValueError(f"UpsertHandle: {len(insert)} insert flags for {n} commands")
        return n

    def clear_input(self):
        """clear_input (input.rs:879-882): drop the commands buffered since the last step."""
        self.pending = []

    def _take(self) -> Batch:
        """This step's commands as one command batch, in order."""
        chunks, self.pending = self.pending, []
        be, comm, s = self.circuit.be, self.circuit.comm, self.schema
        seq = (comm.rank if comm is not None else 0) << self.SEQ_RANK_SHIFT
        out = None
        for c in chunks:
            if c[0] == "rows":
                arr = np.array([[int(x) & _M64 for x in r[0]] for r in c[1]], dtype=np.uint64).reshape(len(c[1]), s.nl)
                b = be.upsert_commands(s, [arr[:, i] for i in range(s.nl)], [r[1] for r in c[1]], seq0=seq)
                n = len(c[1])
            elif c[0] == "host":
                b = be.upsert_commands(s, c[1], c[2], seq0=seq)
                n = len(c[1][0])
            else:
                b = be.upsert_commands(s, c[1], c[3], n=c[2], seq0=seq, on_device=True)
                n = c[2]
            seq += n
            out = b if out is None else be.merge(out, b)
        return out if out is not None else be.batch_empty(upsert_command_schema(s))


class RootCircuit:
    """RootCircuit::build + CircuitHandle::step
    (circuit_builder.rs:1403-1433, 3658-3663)."""

    def __init__(self, backend: Backend | None = None, comm=None):
        if backend is None:
            from .runtime import Runtime  # the CUDA library; raises if unavailable

            backend = Runtime()
        self.be = backend
        self.comm = comm  # parallel.Comm or None (single worker)
        if comm is not None and getattr(comm, "native", None) is None and hasattr(comm, "attach") and comm.world_size > 1:
            comm.attach(backend)   # CUDA backend: the exchange moves into the library (csrc/comm.cu)
        self.nodes: list[Node] = []

    # -- sources -------------------------------------------------------------
    def add_input_zset(self, schema: Schema):
        """add_input_zset / add_input_indexed_zset (operator/input.rs:75-86)."""
        h = InputHandle(self, schema)
        node = Node(self, [], h._take, "input")
        return Stream(self, node, schema), h

    add_input_indexed_zset = add_input_zset

    def add_input_set(self, schema: Schema):
        """add_input_set (operator/input.rs:168-245): an OrdZSet of the schema's lanes (all of them key lanes) fed by
        insert / delete commands with set semantics: inserting a present row and deleting an absent one do nothing.
        Returns (stream, UpsertHandle)."""
        return self._add_upsert(Schema(schema.lanes), is_map=False)

    def add_input_map(self, schema: Schema):
        """add_input_map (operator/input.rs:247-328): an indexed Z-set with the schema's key and value lanes (at
        least one of each) fed by upserts: a key's new value retracts its old one, a delete retracts it.  Returns
        (stream, UpsertHandle)."""
        if schema.nk == 0 or schema.nv == 0:
            raise ValueError(f"add_input_map: a map has key lanes and value lanes, got {schema}")
        return self._add_upsert(schema, is_map=True)

    def _add_upsert(self, schema: Schema, is_map: bool):
        """add_upsert (input.rs:128-166) + Upsert (operator/upsert.rs): the step's command batch, sharded by key, is
        applied to the table's trace, which the stream owns (`stream.table_trace`)."""
        be = self.be
        be.upsert_commands(schema, [np.zeros(0, np.uint64)] * schema.nl)   # the library refuses a bad table now
        h = UpsertHandle(self, schema, is_map)
        cmds = Stream(self, Node(self, [], h._take, "upsert_commands"), upsert_command_schema(schema)).shard()
        table = Spine(be, schema)

        def fn(c: Batch):
            out = be.upsert_delta(c, table)
            table.insert(out)
            return out

        out = cmds._unary(fn, "upsert", schema, True)
        out.table_trace = table
        return out, h

    def add_input_table(self, n_cols: int):
        h = TableHandle()
        node = Node(self, [], h._take, "table")
        return TableStream(self, node, n_cols), h

    def add_source(self, gen: Callable[[], object], schema: Schema | None = None):
        """Generator source (operator/generator.rs): gen() each step."""
        node = Node(self, [], gen, "source")
        return Stream(self, node, schema)

    def step(self):
        for n in self.nodes:
            n.eval()

    @property
    def workers(self):
        return self.comm.world_size if self.comm is not None else 1


class TableStream:
    def __init__(self, circuit, node, n_cols):
        self.circuit, self.node, self.n_cols = circuit, node, n_cols
        self.projs = []   # projections consuming this table, in creation order

    def table_mask(self) -> int:
        """Columns read by any consumer of this table (bit l = column l)."""
        m = 0
        for p in self.projs:
            m |= self.circuit.be.proj_table_mask(p)
        return m

    def flat_map_index(self, proj: Proj) -> "Stream":
        """flat_map_index on the event stream (filter_map.rs:143-152,700-724):
        filter + project + from_tuples, straight from the raw columns.  A fan-out `proj` (`Proj(..., fanout=n)`)
        yields up to n rows per event, from the table and from an upload alike."""
        be = self.circuit.be
        self.projs.append(proj)

        def fn(t):
            if t is None:
                return be.batch_empty(proj.schema)
            kind, cols, w, n = t
            if kind == "upload":
                return be.batch_from_upload(cols, proj)
            return be.batch_from_table(cols, proj, weights=w, n=n, on_device=(kind == "dev"))

        return Stream(self.circuit, Node(self.circuit, [self.node], fn, "flat_map_index"), proj.schema)


class Stream:
    """Stream<RootCircuit, Batch> for Batch in {OrdZSet, OrdIndexedZSet}, or a
    host scalar stream (schema None)."""

    def __init__(self, circuit: RootCircuit, node: Node, schema: Schema | None, sharded=False):
        self.circuit, self.node, self.schema, self.sharded = circuit, node, schema, sharded

    # -- plumbing ------------------------------------------------------------
    def _unary(self, fn, name, schema, sharded=False) -> "Stream":
        return Stream(self.circuit, Node(self.circuit, [self.node], fn, name), schema, sharded)

    def _binary(self, other, fn, name, schema, sharded=False) -> "Stream":
        return Stream(self.circuit, Node(self.circuit, [self.node, other.node], fn, name), schema, sharded)

    def inspect(self, cb: Callable) -> "Stream":
        """inspect (operator/inspect.rs)."""

        def fn(v):
            cb(v)
            return v

        return self._unary(fn, "inspect", self.schema, self.sharded)

    def output(self):
        """OutputHandle: .value after each step."""
        return self.node

    def apply(self, f: Callable) -> "Stream":
        """apply (operator/apply.rs): host function on the stream's value."""
        return self._unary(f, "apply", None)

    # -- linear / stateless --------------------------------------------------
    def index(self, nk: int) -> "Stream":
        """index() (operator/index.rs:128-157): OrdZSet<(K,V)> -> OrdIndexedZSet<K,V>."""
        be = self.circuit.be
        return self._unary(lambda b: be.reindex(b, nk), "index", self.schema.reindex(nk))

    def map_index(self, proj: Proj) -> "Stream":
        """map_index / flat_map_index / map / filter (filter_map.rs:563-577,700-724)."""
        be = self.circuit.be
        return self._unary(lambda b: be.map_index(b, proj), "map_index", proj.schema)

    # the reference's closure-taking variants all lower to one projection + filter in the row language:
    # map / flat_map produce an OrdZSet, map_index / flat_map_index / index_with an OrdIndexedZSet — the output
    # schema of `proj` says which (filter_map.rs:40-215, index.rs:38-62).  A flat_map closure that returns several
    # rows per input row is a fan-out `Proj(..., fanout=n)`; the backend runs it with dbsp_map_index_fanout.
    map = map_index
    flat_map = map_index
    flat_map_index = map_index
    index_with = map_index

    def filter(self, *preds) -> "Stream":
        """filter (operator/filter_map.rs:40-54): keep the rows satisfying every predicate; schema unchanged."""
        from .zset import key, val

        s = self.schema
        ident = [key(i) for i in range(s.nk)] + [val(i) for i in range(s.nv)]
        return self.map_index(Proj(s, ident, list(preds)))

    def sum(self, others: Sequence["Stream"]) -> "Stream":
        """sum (operator/sum.rs:20-40): self + every stream of `others` (aliases allowed)."""
        out = self
        for o in others:
            out = out.plus(o)
        return out

    def neg(self) -> "Stream":
        be = self.circuit.be
        return self._unary(lambda b: be.neg(b), "neg", self.schema, self.sharded)

    def plus(self, other: "Stream") -> "Stream":
        """plus (operator/plus.rs:127-143) = batch merge."""
        be = self.circuit.be
        return self._binary(other, lambda a, b: be.merge(a, b), "plus", self.schema, self.sharded and other.sharded)

    def minus(self, other: "Stream") -> "Stream":
        be = self.circuit.be
        return self._binary(other, lambda a, b: be.merge(a, be.neg(b)), "minus", self.schema)

    def stream_distinct(self) -> "Stream":
        """stream_distinct (operator/distinct.rs:40-52)."""
        be = self.circuit.be
        s = self.shard()
        return s._unary(lambda b: be.stream_distinct(b), "stream_distinct", self.schema, True)

    def stream_join(self, other: "Stream", proj: Proj) -> "Stream":
        """stream_join (operator/join.rs:52-84): stateless Join::eval."""
        be = self.circuit.be
        l, r = self.shard_with(other)
        return l._binary(r, lambda a, b: be.join_batches(a, b, proj), "stream_join", proj.schema)

    def semijoin_stream(self, keys: "Stream") -> "Stream":
        """semijoin_stream (operator/semijoin.rs:38-62)."""
        be = self.circuit.be
        l, r = self.shard(), keys.shard()
        return l._binary(r, lambda a, b: be.semijoin(a, b), "semijoin", Schema(self.schema.lanes), True)

    # -- stateful ------------------------------------------------------------
    def integrate(self) -> "Stream":
        """integrate (operator/integrate.rs): running sum of deltas."""
        be = self.circuit.be
        state = {"acc": None}

        def fn(b):
            state["acc"] = b if state["acc"] is None else be.merge(state["acc"], b)
            return state["acc"]

        return self._unary(fn, "integrate", self.schema, self.sharded)

    def differentiate(self) -> "Stream":
        """differentiate (operator/differentiate.rs): x[t] - x[t-1]."""
        be = self.circuit.be
        state = {"prev": None}

        def fn(b):
            out = b if state["prev"] is None else be.merge(b, be.neg(state["prev"]))
            state["prev"] = b
            return out

        return self._unary(fn, "differentiate", self.schema, self.sharded)

    def join(self, other: "Stream", proj: Proj) -> "Stream":
        """join / join_index / join_generic (operator/join.rs:180-292):
        delta_L |x| trace(R) + delta_R |x| z^-1 trace(L), both sides sharded."""
        be = self.circuit.be
        left, right = self.shard_with(other)
        lt, rt = Spine(be, left.schema), Spine(be, right.schema)

        def fn(dl: Batch, dr: Batch):
            rt.insert(dr)                                            # right.trace()
            o1 = be.join_delta_trace(dl, rt, proj, delta_is_left=True)
            o2 = be.join_delta_trace(dr, lt, proj, delta_is_left=False)  # vs delayed left trace
            lt.insert(dl)                                            # left.trace()
            return be.merge(o1, o2)                                  # left.plus(&right)

        return left._binary(right, fn, "join", proj.schema)

    join_index = join

    def antijoin(self, other: "Stream") -> "Stream":
        """antijoin (operator/join.rs:294-320): the rows of `self` whose key is
        absent from `other` = self - self |x| distinct(other) with the identity
        closure (k, v1).  A row (k, v1, w) gets the weight w·(1 − N(k)), N(k)
        being the number of distinct (k, v2) rows of `other`; so a key with two
        or more of them gives negative weights, as in the reference.

        Keyed streams keep N as a trace of per-key counts and run
        dbsp_antijoin_delta, which never expands a key's values against the
        other side's.  A key-less stream runs the composition above."""
        be = self.circuit.be
        if self.schema.nk == 0 or not be.api.exports("antijoin_delta"):
            return self._antijoin_composed(other)
        left, right = self.shard_with(other)
        a, ib = Spine(be, left.schema), Spine(be, right.schema)   # z^-1 of self's and other's integrals
        nb = _KeyCounts(be, right.schema)

        def fn(da: Batch, db: Batch):
            dnb = nb.step(db, ib)
            ib.insert(db)
            out = be.antijoin_delta(da, a, dnb, nb.trace)
            a.insert(da)
            return out

        return left._binary(right, fn, "antijoin", self.schema, True)   # mark_sharded (join.rs:316)

    def _antijoin_composed(self, other: "Stream") -> "Stream":
        """self - self |x| distinct(other), as join.rs:294-320 composes it: the only antijoin of a key-less stream
        (the join is then a cross product), and the one of a library without dbsp_antijoin_delta."""
        s1 = self.shard()
        s2 = other.distinct().shard()
        nk, nv = self.schema.nk, self.schema.nv
        ident = Proj(self.schema, [key(i) for i in range(nk)] + [lval(i) for i in range(nv)])
        out = s1.minus(s1.join(s2, ident))
        out.sharded = True   # mark_sharded (join.rs:316)
        return out

    def outer_join(self, other: "Stream", f: Proj, fl: Proj, fr: Proj) -> "Stream":
        """outer_join (operator/join.rs:332-360) = join(f) + antijoin(self, other).map(fl) + antijoin(other, self)
        .map(fr): SQL's FULL OUTER JOIN.  `f` is a join closure (key / lval / rval), `fl` a map closure over self's
        rows, `fr` one over other's rows (their values are lval, and rval reads the same lanes); all three have one
        out_schema.  The join's two traces are also the antijoins' traces and the delayed integrals their key
        counts come from, so each input is held once."""
        for name, p in (("f", f), ("fl", fl), ("fr", fr)):
            if p.is_fanout:
                raise ValueError(f"outer_join: {name} is a fan-out closure; an outer join yields one row per match or row")
        if fl.schema != f.schema or fr.schema != f.schema:
            raise ValueError(f"outer_join: f, fl and fr must have one out_schema, have {f.schema}, {fl.schema}, {fr.schema}")
        if self.schema.nk == 0:
            raise ValueError("outer_join: a key-less stream has no key set to count")
        be = self.circuit.be
        left, right = self.shard_with(other)
        lt, rt = Spine(be, left.schema), Spine(be, right.schema)
        na, nb = _KeyCounts(be, left.schema), _KeyCounts(be, right.schema)

        def fn(dl: Batch, dr: Batch):
            # every read sees the state the formula names: the counts and antijoins use z^-1 of the integrals
            dna, dnb = na.step(dl, lt), nb.step(dr, rt)
            ol = be.map_index(be.antijoin_delta(dl, lt, dnb, nb.trace), fl)
            orr = be.map_index(be.antijoin_delta(dr, rt, dna, na.trace), fr)
            rt.insert(dr)                                             # then Stream.join's order
            o1 = be.join_delta_trace(dl, rt, f, delta_is_left=True)
            o2 = be.join_delta_trace(dr, lt, f, delta_is_left=False)
            lt.insert(dl)
            return be.merge(be.merge(o1, o2), be.merge(ol, orr))

        return left._binary(right, fn, "outer_join", f.schema)

    def outer_join_default(self, other: "Stream", f: Proj) -> "Stream":
        """outer_join_default (operator/join.rs:362-386): outer_join with fl = f over a right value of zeros and
        fr = f over a left value of zeros (Default::default() of u64 / i64).  A filter of `f` (its `where`) is part
        of the closure: it holds or not for the matched rows as it does in join(f), and for an unmatched row it is
        evaluated with the missing side's value lanes read as 0, like the output lanes.  The reference's closure has
        no separate filter, so with one this goes beyond it."""
        fl = Proj(f.schema, [_zero_src(o, capi.SRC_RVAL) for o in f.out], [_zero_src(w, capi.SRC_RVAL) for w in f.where])
        fr = Proj(f.schema, [_zero_src(o, capi.SRC_LVAL) for o in f.out], [_zero_src(w, capi.SRC_LVAL) for w in f.where])
        return self.outer_join(other, f, fl, fr)

    def join_incremental(self, other: "Stream", proj: Proj) -> "Stream":
        """join_incremental (operator/join.rs:136-155):
        I(a) |x| I(b) - z^-1(I(a)) |x| z^-1(I(b)), via stateless joins."""
        be = self.circuit.be
        l, r = self.shard(), other.shard()
        st = {"a": None, "b": None}

        def fn(da, db):
            a = da if st["a"] is None else be.merge(st["a"], da)
            b = db if st["b"] is None else be.merge(st["b"], db)
            cur = be.join_batches(a, b, proj)
            if st["a"] is not None:
                cur = be.merge(cur, be.neg(be.join_batches(st["a"], st["b"], proj)))
            st["a"], st["b"] = a, b
            return cur

        return l._binary(r, fn, "join_incremental", proj.schema)

    def aggregate(self, aggregator, local: bool = False) -> "Stream":
        """aggregate (operator/aggregate/mod.rs:204-244): AggregateIncremental
        over stream.trace(), then upsert into the output trace.
        `local=True` skips the shard(): every worker aggregates its own rows —
        the first level of a two-level aggregate for semigroup aggregators
        (MinSemigroup / MaxSemigroup, aggregate/min.rs:17-27), whose partial
        results are then aggregated again after a shard of <= P rows per key."""
        be = self.circuit.be
        if isinstance(aggregator, Fold):
            if local:
                raise ValueError("aggregate(Fold, local=True): Fold is not a semigroup, so per-worker partial folds "
                                 "cannot be combined")
            return self._aggregate_fold(aggregator)
        s = Stream(self.circuit, self.node, self.schema, True) if local else self.shard()
        kind = aggregator.kind
        if kind in (capi.AGG_MAX, capi.AGG_MIN):
            out_schema = s.schema
        else:
            out_schema = Schema(s.schema.key, "u")
        in_tr, out_tr = Spine(be, s.schema), Spine(be, out_schema)

        def fn(d: Batch):
            in_tr.insert(d)
            out = be.aggregate_delta(d, in_tr, out_tr, kind)
            out_tr.insert(out)
            return out

        return s._unary(fn, "aggregate", out_schema, not local)

    def _fold_schema(self, fold: Fold) -> Schema:
        api = self.circuit.be.api
        if not api.exports("aggregate_fold"):
            raise capi.DbspError(f"{api.prefix}aggregate_fold: this library does not export it")
        return Schema(self.schema.key, fold.output.schema.val)

    def _aggregate_fold(self, fold: Fold) -> "Stream":
        be = self.circuit.be
        out_schema = self._fold_schema(fold)
        s = self.shard()
        in_tr, out_tr = Spine(be, s.schema), Spine(be, out_schema)

        def fn(d: Batch):
            in_tr.insert(d)
            out = be.aggregate_fold(d, in_tr, out_tr, fold)
            out_tr.insert(out)
            return out

        return s._unary(fn, "aggregate", out_schema, True)

    def stream_aggregate(self, aggregator) -> "Stream":
        """stream_aggregate (operator/aggregate/mod.rs:172-196): Aggregate::eval
        (:362-376) — the aggregate of every key of *this step's* batch with
        weight +1; no state.  Runs the same kernels as `aggregate` on a trace
        holding only the batch and an empty output trace."""
        be = self.circuit.be
        s = self.shard()
        if isinstance(aggregator, Fold):
            out_schema = self._fold_schema(aggregator)

            def run(d, tin, tout):
                return be.aggregate_fold(d, tin, tout, aggregator)
        else:
            kind = aggregator.kind
            out_schema = s.schema if kind in (capi.AGG_MAX, capi.AGG_MIN) else Schema(s.schema.key, "u")

            def run(d, tin, tout):
                return be.aggregate_delta(d, tin, tout, kind)

        def fn(d: Batch):
            if len(d) == 0:
                return be.batch_empty(out_schema)
            tin, tout = Spine(be, s.schema), Spine(be, out_schema)
            tin.insert(d)
            return run(d, tin, tout)

        return s._unary(fn, "stream_aggregate", out_schema, True)

    def weigh(self, f, mode=capi.WEIGH_LINEAR) -> "Stream":
        """weigh (operator/aggregate/mod.rs:285-323)."""
        be = self.circuit.be
        sch = Schema(self.schema.key + ("u" if mode == capi.WEIGH_AVG else ""), "")
        return self._unary(lambda b: be.weigh(b, f, mode), "weigh", sch, self.sharded)

    def aggregate_linear(self, f) -> "Stream":
        """aggregate_linear (aggregate/mod.rs:253-273) = weigh(f).aggregate(WeightedCount)."""
        be = self.circuit.be
        w = self.weigh(f).shard()   # weigh first (linear): only one row per key crosses the exchange
        out_schema = Schema(self.schema.key, "i")
        in_tr, out_tr = Spine(be, w.schema), Spine(be, out_schema)

        def fn(d: Batch):
            in_tr.insert(d)
            out = be.aggregate_delta(d, in_tr, out_tr, capi.AGG_WCOUNT)
            out_tr.insert(out)
            return out

        return w._unary(fn, "aggregate_linear", out_schema, True)

    def average(self, f) -> "Stream":
        """average (operator/aggregate/average.rs:227-246): aggregate_linear
        with the (sum,count) pair weight, then apply_average (:266-307) —
        truncating signed division of the value column.  The pair weight is
        carried as two rows (K,0)->sum and (K,1)->count of an OrdZSet (see
        include/dbsp_b200.h, DBSP_AGG_WCOUNT2).  Unlike apply_average the
        result is re-consolidated, which only removes +1/-1 pairs that the
        reference's downstream map/from_tuples would cancel anyway."""
        be = self.circuit.be
        # weigh first (linear): <= 2 rows per key cross the exchange; shard on K only so that
        # the (K,0) and (K,1) rows of a key meet on one worker (index() is a zero-copy view)
        nk0 = self.schema.nk
        w = self.weigh(f, capi.WEIGH_AVG).index(nk0).shard().index(nk0 + 1)
        pair_schema = Schema(self.schema.key, "ii")
        out_schema = Schema(self.schema.key, "i")
        in_tr, out_tr = Spine(be, w.schema), Spine(be, pair_schema)
        nk = self.schema.nk
        # a key whose count sums to 0 (its sum need not) has no average: no row, where the reference panics
        avg = Proj(out_schema, [key(i) for i in range(nk)] + [lval(0) // lval(1)], where=[lval(1).ne(0)])

        def fn(d: Batch):
            in_tr.insert(d)
            out = be.aggregate_delta(d, in_tr, out_tr, capi.AGG_WCOUNT2)
            out_tr.insert(out)
            return be.map_index(out, avg)

        return w._unary(fn, "average", out_schema, True)

    def distinct(self) -> "Stream":
        """distinct (operator/distinct.rs:64-106): DistinctIncrementalTotal
        against the delayed integral of the sharded input."""
        be = self.circuit.be
        s = self.shard()
        integral = Spine(be, s.schema)

        def fn(d: Batch):
            out = be.distinct_delta(d, integral)
            integral.insert(d)
            return out

        return s._unary(fn, "distinct", s.schema, True)

    def window(self, bounds: "Stream") -> "Stream":
        """window (operator/time_series/window.rs:75-86): the trace is delayed
        and truncated below the previous lower bound (operator/trace.rs:578-605)."""
        be = self.circuit.be
        trace = Spine(be, self.schema)
        st = {"prev": None}
        nk = self.schema.nk

        def norm(b):
            lo, hi = b
            lo = tuple(lo) if isinstance(lo, (tuple, list)) else (lo,)
            hi = tuple(hi) if isinstance(hi, (tuple, list)) else (hi,)
            assert len(lo) == nk and len(hi) == nk
            return lo, hi

        def fn(d: Batch, b):
            cur = norm(b)
            out = be.window_delta(trace, d, st["prev"], cur)
            trace.insert(d)
            trace.truncate_keys_below(cur[0])
            st["prev"] = cur
            return out

        out = self._binary(bounds, fn, "window", self.schema, self.sharded)
        out.window_trace = trace   # the bounded trace of the operator (window.rs:454-486 asserts that it stays small)
        return out

    def watermark_monotonic(self, f: Callable[[int], int]) -> "Stream":
        """watermark_monotonic (operator/time_series/watermark.rs:33-74): max of
        the previous watermark and f(last key of the batch); all-reduced (max)
        across workers."""
        comm = self.circuit.comm
        st = {"wm": 0}

        def fn(b: Batch):
            k = b.last_key()
            if k is not None:
                st["wm"] = max(st["wm"], f(k[0] if len(k) == 1 else k))
            if comm is not None and comm.world_size > 1:
                st["wm"] = comm.allreduce_max(st["wm"])
            return st["wm"]

        return self._unary(fn, "watermark_monotonic", None)

    # -- time series ---------------------------------------------------------
    def partitioned_rolling_aggregate(self, aggregator, rng: RelRange) -> "Stream":
        """partitioned_rolling_aggregate (operator/time_series/rolling_aggregate.rs:235-249): the stream is indexed by
        the partition key PK, value lane 0 is the timestamp TS and the other value lanes are V.  For every (pk, ts)
        with a row of positive weight, the output holds (pk, (ts, some, agg..)): `agg` aggregates the partition's rows
        whose ts' lies in rng.range_of(ts), `some` is 0 (and agg 0) when none does.  `aggregator` is Max, Min (over V)
        or Linear(f).  The stream is sharded by PK first.  The operator's traces are the stream's `rolling_in_trace` and
        `rolling_out_trace`."""
        return self._rolling(self, aggregator, rng)

    def partitioned_rolling_aggregate_linear(self, f: Proj, rng: RelRange) -> "Stream":
        """partitioned_rolling_aggregate_linear (rolling_aggregate.rs:367-385) = the rolling aggregate of Linear(f)."""
        return self._rolling(self, Linear(f), rng)

    def partitioned_rolling_aggregate_with_watermark(self, watermark: "Stream", partition: Proj, aggregator,
                                                     rng: RelRange) -> "Stream":
        """partitioned_rolling_aggregate_with_watermark (rolling_aggregate.rs:155-220): the stream is indexed by the
        timestamp (one key lane) and `partition` maps its value to (pk.., v..) (its key lanes are PK, its value lanes
        V).  The watermark bounds the state: the input is windowed to [lower, max), lower = the start of the range
        [from - to, Before(0)] of the watermark, and the output trace drops times below lower after each step.  Both
        traces and the window's are exposed on the result (`rolling_in_trace`, `rolling_out_trace`, `window_trace`),
        and `rolling_lower()` is the current lower bound."""
        if self.schema.nk != 1:
            raise ValueError(f"partitioned_rolling_aggregate_with_watermark: the stream is indexed by the timestamp "
                             f"alone, has {self.schema.nk} key lanes")
        ts = self.schema.key
        signed = ts == "i"
        lo_ts, hi_ts = (-(1 << 63), (1 << 63) - 1) if signed else (0, (1 << 64) - 1)
        shifted = RelRange(rng.frm.sub(rng.to, signed), Before(0))
        st = {"lower": lo_ts}

        def bounds(wm):
            r = shifted.range_of(wm, signed)
            st["lower"] = lo_ts if r is None else r[0]
            return st["lower"], hi_ts

        window = self.window(watermark.apply(bounds))
        pnk = partition.schema.nk
        by_pk = Proj(Schema(partition.schema.key, ts + partition.schema.val),
                     partition.out[:pnk] + [key(0)] + partition.out[pnk:], partition.where)
        out = self.map_index(by_pk)._rolling(window.map_index(by_pk), aggregator, rng, lambda: st["lower"])
        out.window_trace = window.window_trace
        out.rolling_lower = lambda: st["lower"]
        return out

    def _rolling(self, win: "Stream", aggregator, rng: RelRange, lower: Callable[[], int] | None = None) -> "Stream":
        """PartitionedRollingAggregate (rolling_aggregate.rs:286-359): the delta is `self`, the input trace integrates
        `win` (self, or its windowed form), the output trace holds the operator's past outputs; `lower`, when given,
        truncates the output trace's times below it after each step."""
        be = self.circuit.be
        if not be.api.exports("rolling_aggregate"):
            raise capi.DbspError(f"{be.api.prefix}rolling_aggregate: this library does not export it")
        kind, f = _rolling_kind(aggregator)
        s = self.schema
        if s.nv == 0:
            raise ValueError("partitioned_rolling_aggregate: the stream has no value lanes; value lane 0 is the timestamp")
        agg = f.schema.val if f is not None else s.val[1:]
        out_schema = Schema(s.key, s.val[0] + "u" + agg)
        d = self.shard()
        w = d if win is self else win.shard()
        in_tr, out_tr = Spine(be, s), Spine(be, out_schema)

        def fn(dd: Batch, wd: Batch):
            in_tr.insert(wd)
            out = be.rolling_aggregate(dd, in_tr, out_tr, rng, kind, f)
            out_tr.insert(out)
            if lower is not None:
                out_tr.truncate_values_below([lower()] + [0] * (out_schema.nv - 1))
            return out

        node = Node(self.circuit, [d.node, w.node], fn, "partitioned_rolling_aggregate")
        out = Stream(self.circuit, node, out_schema, True)
        out.rolling_in_trace, out.rolling_out_trace = in_tr, out_tr
        return out

    # -- communication -------------------------------------------------------
    def shard(self) -> "Stream":
        """shard (operator/communication/shard.rs:89-162): hash-partition by
        key, all-to-all, merge at the receiver.  Identity with one worker
        (shard.rs:111-114) or when already sharded."""
        comm = self.circuit.comm
        if comm is None or comm.world_size == 1 or self.sharded:
            return Stream(self.circuit, self.node, self.schema, True)
        be = self.circuit.be
        return self._unary(lambda b: comm.shard(be, b), "shard", self.schema, True)

    def shard_with(self, other: "Stream") -> tuple["Stream", "Stream"]:
        """shard() of both inputs of a binary operator (join.rs:265-266) in ONE
        exchange round: same result as (self.shard(), other.shard())."""
        comm = self.circuit.comm
        if comm is None or comm.world_size == 1 or self.sharded or other.sharded:
            return self.shard(), other.shard()
        be = self.circuit.be
        pair = Node(self.circuit, [self.node, other.node], lambda a, b: comm.shard_many(be, [a, b]), "shard2")
        left = Stream(self.circuit, Node(self.circuit, [pair], lambda t: t[0], "shard2.0"), self.schema, True)
        right = Stream(self.circuit, Node(self.circuit, [pair], lambda t: t[1], "shard2.1"), other.schema, True)
        return left, right

    def gather(self, root: int = 0) -> "Stream":
        """gather (operator/communication/gather.rs:41-103)."""
        comm = self.circuit.comm
        if comm is None or comm.world_size == 1:
            return self
        be = self.circuit.be
        return self._unary(lambda b: comm.gather(be, b, root), "gather", self.schema)
