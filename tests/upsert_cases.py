"""Cases of the set and map input tables (`add_input_set`, `add_input_map`: dbsp_upsert_commands + dbsp_upsert_delta),
shared by the oracle and CUDA tests.

The model is not incremental: a Python dict (a set is a dict of keys to ()) that applies each step's commands in
order; a step's expected output is the Z-set difference of the states before and after it.  Every case runs its
circuit on `be` against the model, and, given `ref`, on `ref` as well, bit for bit against `be`."""
import json
import os

import numpy as np

from dbsp_b200 import RootCircuit, Schema, Spine
from dbsp_b200._capi import DbspError
from dbsp_b200.zset import upsert_command_schema
from horizon_cases import PAIRS
from parity_util import assert_batches_equal

HERE = os.path.dirname(os.path.abspath(__file__))
M64 = (1 << 64) - 1
GOLDEN = os.path.join(HERE, "golden", "upsert_input.json")
DOC_NAMES = {"foo": 1, "bar": 2, "baz": 3}
GARBAGE = 0xDEAD_BEEF_0BAD_F00D   # value lanes of a delete given as columns: ignored


def norm(types, t):
    """Lanes as Batch.rows() gives them: i64 lanes signed, u64 lanes unsigned."""
    out = []
    for ty, x in zip(types, t):
        x = int(x) & M64
        out.append(x - (1 << 64) if ty == "i" and x >= 1 << 63 else x)
    return tuple(out)


def as_tuple(x):
    return tuple(x) if isinstance(x, (tuple, list)) else (x,)


class Model:
    """The table as a dict key -> value tuple, commands applied in order."""

    def __init__(self, schema, is_map):
        self.s, self.is_map, self.state = schema, is_map, {}

    def rows(self):
        return {k + v: 1 for k, v in self.state.items()}

    def apply(self, cmds):
        old = self.rows()
        s = self.s
        for k, v in cmds:
            k = norm(s.key, as_tuple(k))
            if self.is_map and v is not None:
                self.state[k] = norm(s.val, as_tuple(v))
            elif not self.is_map and v:
                self.state[k] = ()
            else:
                self.state.pop(k, None)
        return zdiff(self.rows(), old)


def zdiff(new, old):
    out = dict(new)
    for r, w in old.items():
        out[r] = out.get(r, 0) - w
    return {r: w for r, w in out.items() if w != 0}


def zdict(b):
    return {r[:-1]: r[-1] for r in b.rows()}


# ---- feeding a handle ----------------------------------------------------------------------------------------------
def columns(schema, is_map, cmds):
    """Commands as (u64 columns of the table's lanes, insert flags); a delete's value lanes hold garbage."""
    n = len(cmds)
    cols = [np.zeros(n, np.uint64) for _ in range(schema.nl)]
    ins = np.zeros(n, np.uint8)
    for i, (k, v) in enumerate(cmds):
        k = as_tuple(k)
        insert = (v is not None) if is_map else bool(v)
        vals = as_tuple(v) if (is_map and insert) else (GARBAGE,) * schema.nv
        for l, x in enumerate(k + vals):
            cols[l][i] = int(x) & M64
        ins[i] = insert
    return cols, ins


class Device:
    """Resident columns for append_device: CUDA tensors on the GPU; on the oracle, whose device columns are host
    memory, the numpy arrays themselves."""

    def __init__(self, be):
        self.be, self.keep = be, []

    def put(self, arr):
        if self.be.name == "oracle":
            a = np.ascontiguousarray(arr)
            self.keep.append(a)
            return a.ctypes.data
        import torch

        t = torch.from_numpy(np.ascontiguousarray(arr).view(np.int64 if arr.dtype == np.uint64 else np.uint8)).cuda()
        self.keep.append(t)
        return int(t.data_ptr())


def feed(h, cmds, mode, dev=None):
    """mode: append | push | columns | device | mixed (rows, columns and device appends in turn)."""
    s, is_map = h.schema, h.is_map
    if mode == "append":
        h.append(list(cmds))
    elif mode == "push":
        for k, v in cmds:
            h.push(k, v)
    elif mode == "columns":
        cols, ins = columns(s, is_map, cmds)
        h.append_columns(cols, ins)
    elif mode == "device":
        cols, ins = columns(s, is_map, cmds)
        h.append_device([dev.put(c) for c in cols], len(cmds), dev.put(ins))
    else:
        parts = np.array_split(np.arange(len(cmds)), 7)
        for j, idx in enumerate(parts):
            feed(h, [cmds[i] for i in idx], ("push", "columns", "device", "append")[j % 4], dev)


class Run:
    """One set / map input on one backend: its circuit, output and handle."""

    def __init__(self, be, schema, is_map):
        self.be, self.c = be, RootCircuit(be)
        self.stream, self.h = self.c.add_input_map(schema) if is_map else self.c.add_input_set(schema)
        self.out = self.stream.output()
        self.dev = Device(be)

    def step(self, cmds, mode):
        feed(self.h, cmds, mode, self.dev)
        self.c.step()
        self.dev.keep = []
        return self.out.value


def run_steps(be, ref, schema, is_map, steps, mode="append", check_trace=False, what=""):
    """Every step against the model (and `ref`, bit for bit); with check_trace, the consolidated table trace too."""
    model = Model(Schema(schema.lanes) if not is_map else schema, is_map)
    runs = [Run(b, schema, is_map) for b in ((be, ref) if ref is not None else (be,))]
    for t, cmds in enumerate(steps):
        exp = model.apply(cmds)
        outs = [r.step(cmds, mode) for r in runs]
        assert zdict(outs[0]) == exp, f"{what} step {t} ({mode})"
        if ref is not None:
            assert_batches_equal(outs[0], outs[1], f"{what} step {t} ({mode}) vs oracle")
        if check_trace:
            assert zdict(runs[0].stream.table_trace.consolidate()) == model.rows(), f"{what} step {t}: trace"
    return runs


# ---- the reference's literals --------------------------------------------------------------------------------------
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def _literal(be, ref, is_map, inputs, outputs, schema, what):
    for mode in ("append", "push"):
        model = Model(schema, is_map)
        runs = [Run(b, schema, is_map) for b in ((be, ref) if ref is not None else (be,))]
        for t, (cmds, out) in enumerate(zip(inputs, outputs)):
            cmds = [(k, v) for k, v in cmds]
            exp = {norm(schema.lanes, r[:-1]): r[-1] for r in out}
            assert model.apply(cmds) == exp, f"{what}: the model disagrees with the reference at step {t}"
            got = [r.step(cmds, mode) for r in runs]
            assert zdict(got[0]) == exp, f"{what} step {t} ({mode})"
            if ref is not None:
                assert_batches_equal(got[0], got[1], f"{what} step {t} ({mode}) vs oracle")


def run_golden_set(be, ref=None):
    g = golden()
    _literal(be, ref, False, g["input_set_updates"], g["output_set_updates"], Schema("u"), "set_test")


def run_golden_map(be, ref=None):
    g = golden()
    _literal(be, ref, True, g["input_map_updates"], g["output_map_updates"], Schema("u", "u"), "map_test")


def run_doc_tables(be, ref=None):
    g = golden()
    name = lambda x: DOC_NAMES.get(x, x) if isinstance(x, str) else x   # noqa: E731
    d = g["doc_set"]
    ins = [[(name(k), b) for k, b in step] for step in d["input"]]
    outs = [[[name(x) for x in r] for r in step] for step in d["output"]]
    _literal(be, ref, False, ins, outs, Schema("u"), "add_input_set doc table")
    d = g["doc_map"]
    ins = [[(k, None if v is None else name(v)) for k, v in step] for step in d["input"]]
    outs = [[[name(x) for x in r] for r in step] for step in d["output"]]
    _literal(be, ref, True, ins, outs, Schema("u", "u"), "add_input_map doc table")


# ---- order -----------------------------------------------------------------------------------------------------------
def run_order(be, ref=None):
    ms = Schema("u", "u")
    steps = [
        [(1, 10), (2, 20), (3, 30)],
        [(1, 11), (1, None)],                  # insert then delete: the key is gone
        [(2, None), (2, 21)],                  # delete then insert: overwritten
        [(3, 30)],                             # the same value re-inserted: nothing
        [(9, None), (1, None)],                # deletes of absent keys: nothing
        [(3, 31), (3, 30)],                    # back to the current value: nothing
        [],                                    # an empty step
        [(4, 40), (4, 41), (4, 40), (2, 21)],
    ]
    for mode in ("append", "push", "columns", "device", "mixed"):
        run_steps(be, ref, ms, True, steps, mode, check_trace=True, what="order")
    set_steps = [[(1, True), (1, False)], [(2, False), (2, True)], [(2, True)], [(7, False)], [(2, False), (2, True), (2, False)]]
    for mode in ("append", "push", "columns", "device", "mixed"):
        run_steps(be, ref, Schema("u"), False, set_steps, mode, check_trace=True, what="order set")


def run_one_hot_key(be, ref=None):
    """One key with 70 000 commands in a step, between other keys; the last is an insert, then a delete."""
    rng = np.random.default_rng(7)
    ms = Schema("i", "u")
    for last in (123456, None):
        hot = [(-5, int(v)) if v % 9 else (-5, None) for v in rng.integers(0, 1 << 40, 70_000)]
        hot[-1] = (-5, last)
        steps = [[(k, k) for k in range(-20, 20)], [(k, 2 * k) for k in range(-20, -5)] + hot + [(k, 3 * k) for k in range(-4, 20)]]
        for mode in ("columns", "mixed"):
            run_steps(be, ref, ms, True, steps, mode, check_trace=True, what=f"hot key, last {last}")


def run_split_appends(be, ref=None):
    """A step's commands over several appends of every kind keep their order, and equal one append."""
    rng = np.random.default_rng(11)
    ms = Schema("uu", "i")
    steps = []
    for t in range(6):
        keys = rng.integers(0, 40, (3000, 2))
        steps.append([((int(a), int(b)), None if rng.random() < 0.2 else int(rng.integers(-9, 9))) for a, b in keys])
    runs = run_steps(be, ref, ms, True, steps, "mixed", check_trace=True, what="split appends")
    whole = run_steps(be, None, ms, True, steps, "columns", what="one append")
    assert_batches_equal(runs[0].stream.table_trace.consolidate(), whole[0].stream.table_trace.consolidate(), "split vs whole")


def run_clear_input(be, ref=None):
    r = Run(be, Schema("u", "u"), True)
    r.h.push(1, 1)
    r.h.append_columns([np.array([2], np.uint64), np.array([2], np.uint64)])
    r.h.clear_input()
    r.h.push(3, 3)
    r.c.step()
    assert zdict(r.out.value) == {(3, 3): 1}


# ---- shapes ----------------------------------------------------------------------------------------------------------
def random_steps(rng, schema, is_map, n_steps, n, key_range, full=False):
    steps = []
    for _ in range(n_steps):
        cmds = []
        for _ in range(n):
            k = tuple(int(x) for x in (rng.integers(0, 1 << 63, schema.nk) * 2 + rng.integers(0, 2, schema.nk)
                                        if full else rng.integers(-key_range, key_range, schema.nk)))
            if not is_map:
                cmds.append((k, bool(rng.random() < 0.6)))
            elif rng.random() < 0.25:
                cmds.append((k, None))
            else:
                cmds.append((k, tuple(int(x) for x in rng.integers(-3, 3, schema.nv))))
        steps.append(cmds)
    return steps


def run_shapes(be, ref=None):
    rng = np.random.default_rng(3)
    for L in range(1, 8):
        s = Schema("".join(rng.choice(["u", "i"], L)))
        run_steps(be, ref, s, False, random_steps(rng, s, False, 4, 400, 6), "columns", True, f"set of {L} lanes")
    for nk in range(1, 7):
        s = Schema("".join(rng.choice(["u", "i"], nk)), "".join(rng.choice(["u", "i"], 1 if nk == 6 else 2)))
        run_steps(be, ref, s, True, random_steps(rng, s, True, 4, 400, 6), "columns", True, f"map {s}")
    s = Schema("i", "i")   # negative keys and values
    run_steps(be, ref, s, True, random_steps(rng, s, True, 5, 2000, 1 << 62), "mixed", True, "i64 lanes")


def run_wide_keys(be, ref=None):
    """Keys of three full-range u64 lanes: wider than the two-word packed sort key.  Keys repeat across steps."""
    rng = np.random.default_rng(5)
    s = Schema("uuu", "u")
    pool = random_steps(rng, s, True, 1, 3000, 0, full=True)[0]
    keys = [k for k, _ in pool]
    steps = []
    for t in range(5):
        idx = rng.integers(0, len(keys), 4000)
        steps.append([(keys[i], None if rng.random() < 0.2 else (int(rng.integers(0, 1 << 63)) * 2,)) for i in idx])
    run_steps(be, ref, s, True, steps, "columns", True, "wide keys")
    run_steps(be, ref, Schema("uuu"), False, [[(keys[i], bool(i % 3)) for i in rng.integers(0, len(keys), 4000)] for _ in range(3)],
              "columns", True, "wide set")


def run_insert_none(be, ref=None):
    """append_columns without flags: a bulk load in which every command inserts."""
    s = Schema("u", "u")
    n = 5000
    model = Model(s, True)
    runs = [Run(b, s, True) for b in ((be, ref) if ref is not None else (be,))]
    for t in range(3):
        k = np.arange(n, dtype=np.uint64) * 3 % 7001
        v = np.full(n, t, np.uint64)
        exp = model.apply([(int(a), int(b)) for a, b in zip(k, v)])
        for r in runs:
            r.h.append_columns([k, v])
            r.c.step()
        assert zdict(runs[0].out.value) == exp, f"insert=None step {t}"
        if ref is not None:
            assert_batches_equal(runs[0].out.value, runs[1].out.value, f"insert=None step {t} vs oracle")


# ---- trace states ----------------------------------------------------------------------------------------------------
def regime_steps(regime, pair, n_steps=64, seed=0):
    """Commands on the schema of a horizon pair's left input, key ids mapped onto its key lanes.
    growth: fresh keys every step and a few overwrites; churn: a fixed key range with inserts, overwrites and
    deletes; hot: a handful of keys taking thousands of commands per step over a churning background."""
    rng = np.random.default_rng(seed)
    s = pair.sl
    steps = []
    for t in range(n_steps):
        if regime == "growth":
            kid = np.concatenate([np.arange(t * 400, (t + 1) * 400), rng.integers(0, (t + 1) * 400, 40)])
            dele = rng.random(len(kid)) < 0.02
        elif regime == "churn":
            kid = rng.integers(-3000, 3000, 1500)
            dele = rng.random(len(kid)) < 0.3
        else:
            kid = np.concatenate([rng.integers(0, 4, 4000), rng.integers(-2000, 2000, 500)])
            dele = rng.random(len(kid)) < 0.15
        kc = pair.key_cols(kid)
        vals = [rng.integers(-50 if ty == "i" else 0, 50, len(kid)) for ty in s.val]
        cmds = []
        for i in range(len(kid)):
            k = tuple(int(c[i]) for c in kc)
            cmds.append((k, None if dele[i] else tuple(int(v[i]) for v in vals)))
        steps.append(cmds)
    return s, steps


def run_trace_states(be, ref=None):
    for pair_name, pair in PAIRS.items():
        for regime in ("growth", "churn", "hot"):
            s, steps = regime_steps(regime, pair)
            runs = run_steps(be, ref, s, True, steps, "columns", check_trace=True, what=f"{regime} {pair_name}")
            _, nb = runs[0].stream.table_trace.stats()
            assert nb >= 2, f"{regime} {pair_name}: the table trace ended with {nb} batch(es)"


def run_weights(be, ref=None):
    """A row of weight 3 inserted into the table trace is retracted by -3 at the key's next command; a set's re-insert
    of such a row gives 1 - 3."""
    for is_map, s, row, cmd, exp in ((True, Schema("u", "u"), (5, 50), (5, 51), {(5, 50): -3, (5, 51): 1}),
                                     (True, Schema("u", "u"), (5, 50), (5, None), {(5, 50): -3}),
                                     (False, Schema("u"), (5,), (5, True), {(5,): -2})):
        got = []
        for b in ((be, ref) if ref is not None else (be,)):
            r = Run(b, s, is_map)
            r.stream.table_trace.insert(b.batch_from_rows(s, [row + (3,)]))
            r.step([cmd], "append")
            got.append(r.out.value)
            assert zdict(got[-1]) == exp, (b.name, cmd)
            assert zdict(r.stream.table_trace.consolidate()) == zdiff(exp, {row: -3}), (b.name, cmd)
        if ref is not None:
            assert_batches_equal(got[0], got[1], f"weight 3, {cmd}")


def run_save_load(be, tmp_path, ref=None):
    """Save the table trace mid-sequence, load it into a new trace, continue both: the same outputs."""
    s, steps = regime_steps("churn", PAIRS["iu_uiu"], 16, seed=9)
    a = Spine(be, s)
    outs_a = []
    b = None
    for t, cmds in enumerate(steps):
        cols, ins = columns(s, True, cmds)
        cb = be.upsert_commands(s, cols, ins, seq0=0)
        if t == 8:
            path = os.path.join(str(tmp_path), f"upsert_{be.name}.spine")
            a.save(path)
            b = Spine.load(be, path, s)
        oa = be.upsert_delta(cb, a)
        a.insert(oa)
        if b is not None:
            ob = be.upsert_delta(cb, b)
            b.insert(ob)
            assert_batches_equal(oa, ob, f"step {t} after the reload")
        outs_a.append(oa)
    assert_batches_equal(a.consolidate(), b.consolidate(), "traces after the reload")


# ---- refusals ----------------------------------------------------------------------------------------------------
def run_refusals(be):
    """One refusal per valid_upsert rule at the ABI (DBSP_ERR_INVALID, a text naming the call and the rule), and the
    Python refusals."""
    import ctypes as C

    api = be.api
    out = C.c_void_p()
    col = np.zeros(4, np.uint64)
    cols = (C.c_void_p * 8)(*([col.ctypes.data] * 8))

    def refused(call, args, text):
        rc = getattr(api, "_" + call)(*args)
        msg = api._last_error().decode()
        assert rc == 1 and call in msg and text in msg, (call, rc, msg)
        assert not out.value

    ms = Schema("u", "u")
    refused("upsert_commands", (be.ctx, None, cols, None, 4, 0, 0, C.byref(out)), "table is NULL")
    refused("upsert_commands", (be.ctx, C.byref(ms.c()), cols, None, 4, 0, 0, None), "out is NULL")
    refused("upsert_commands", (None, C.byref(ms.c()), cols, None, 4, 0, 0, C.byref(out)), "ctx is NULL")
    refused("upsert_commands", (be.ctx, C.byref(ms.c()), None, None, 4, 0, 0, C.byref(out)), "cols is NULL")
    refused("upsert_commands", (be.ctx, C.byref(Schema("", "uu").c()), cols, None, 4, 0, 0, C.byref(out)), "no key lanes")
    refused("upsert_commands", (be.ctx, C.byref(Schema("uuuu", "uuuu").c()), cols, None, 4, 0, 0, C.byref(out)), "at most 7")
    refused("upsert_commands", (be.ctx, C.byref(ms.c()), cols, None, 4, (1 << 63) - 3, 0, C.byref(out)), "exceeds 2^63")
    assert api._upsert_commands(be.ctx, C.byref(ms.c()), cols, None, 4, (1 << 63) - 4, 0, C.byref(out)) == 0   # the last fits
    be.api._batch_free(out.value)
    out.value = None
    tr = Spine(be, ms)
    good = be.upsert_commands(ms, [col, col])
    refused("upsert_delta", (be.ctx, None, tr.h, C.byref(out)), "cmds is NULL")
    refused("upsert_delta", (be.ctx, good.h, None, C.byref(out)), "table is NULL")
    refused("upsert_delta", (be.ctx, good.h, tr.h, None), "out is NULL")
    keyless, wide = Spine(be, Schema("", "uu")), Spine(be, Schema("uuuu", "uuuu"))
    refused("upsert_delta", (be.ctx, good.h, keyless.h, C.byref(out)), "no key lanes")
    refused("upsert_delta", (be.ctx, good.h, wide.h, C.byref(out)), "at most 7")
    bads = [be.batch_empty(Schema(k, v)) for k, v in (("u", "uuu"), ("u", "u"), ("u", "iu"), ("i", "uu"), ("uu", "u"))]
    for bad in bads:
        refused("upsert_delta", (be.ctx, bad.h, tr.h, C.byref(out)), "cmds must have the table's key lanes")
    assert be.upsert_delta(good, tr).schema == ms


def run_python_refusals(be):
    import pytest

    c = RootCircuit(be)
    _, hs = c.add_input_set(Schema("uu"))
    _, hm = c.add_input_map(Schema("u", "ii"))
    for h, k, v in ((hs, 1, True), (hs, (1, 2), 1), (hs, (1, 2, 3), True), (hs, (1, "x"), True), (hs, (True, 2), True),
                    (hm, 1, (1,)), (hm, 1, 5), (hm, (1, 2), (1, 2)), (hm, 1, True), (hm, 1, (1, 2, 3))):
        with pytest.raises(ValueError):
            h.push(k, v)
        with pytest.raises(ValueError):
            h.append([(k, v)])
    assert hs.pending == [] and hm.pending == []
    with pytest.raises(ValueError):
        hm.append_columns([np.zeros(2, np.uint64)] * 2)
    with pytest.raises(ValueError):
        hm.append_columns([np.zeros(2, np.uint64), np.zeros(3, np.uint64), np.zeros(2, np.uint64)])
    with pytest.raises(ValueError):
        hm.append_columns([np.zeros(2, np.uint64)] * 3, insert=[1])
    with pytest.raises(ValueError):
        hm.append_device([0, 0], 2)
    with pytest.raises(ValueError):
        c.add_input_map(Schema("uu"))
    with pytest.raises(ValueError):
        c.add_input_map(Schema("", "uu"))
    with pytest.raises(DbspError, match="at most 7"):
        c.add_input_set(Schema("uuuuuuuu"))
    with pytest.raises(DbspError, match="at most 7"):
        c.add_input_map(Schema("uuuu", "uuuu"))
    with pytest.raises(DbspError, match="exceeds 2"):
        be.upsert_commands(Schema("u"), [np.zeros(2, np.uint64)], seq0=(1 << 63) - 1)
    with pytest.raises(DbspError, match="cmds must have"):
        be.upsert_delta(be.batch_empty(Schema("u", "u")), Spine(be, Schema("u", "u")))


def run_plain_oracle_lacks(oracle):
    import pytest

    for add in ("add_input_set", "add_input_map"):
        with pytest.raises(DbspError, match="orc_upsert_commands: this library does not export it"):
            getattr(RootCircuit(oracle), add)(Schema("u", "u"))


def run_command_batch(be, ref=None):
    """dbsp_upsert_commands itself: the rows, ordered by (key, command word), a delete's values 0."""
    s = Schema("i", "u")
    k = np.array([3, -1, 3, 2, -1], np.int64)
    v = np.array([7, 8, 9, 10, 11], np.uint64)
    b = be.upsert_commands(s, [k, v], [1, 0, 0, 1, 1], seq0=100)
    assert b.schema == upsert_command_schema(s) == Schema("i", "uu")
    assert b.rows() == [(-1, 202, 0, 1), (-1, 209, 11, 1), (2, 207, 10, 1), (3, 201, 7, 1), (3, 204, 0, 1)]
    if ref is not None:
        assert_batches_equal(b, ref.upsert_commands(s, [k, v], [1, 0, 0, 1, 1], seq0=100), "command batch vs oracle")


ALL_CASES = {
    "golden_set": run_golden_set, "golden_map": run_golden_map, "doc_tables": run_doc_tables, "order": run_order,
    "one_hot_key": run_one_hot_key, "split_appends": run_split_appends, "clear_input": run_clear_input,
    "shapes": run_shapes, "wide_keys": run_wide_keys, "insert_none": run_insert_none, "trace_states": run_trace_states,
    "weights": run_weights, "command_batch": run_command_batch,
}


# ---- scale (GPU) -------------------------------------------------------------------------------------------------
def scale_steps(rng, n_live, n, steps):
    """A bulk load of n_live keys (insert=None), then `steps` steps of n commands: a third fresh inserts, a third
    overwrites of live keys, the rest deletes (some of absent keys), shuffled."""
    k0 = rng.permutation(np.arange(n_live, dtype=np.uint64) * 2 + 1)
    yield [k0, k0 * 7, k0 & 1023], None
    nxt = n_live
    for _ in range(steps):
        a = n // 3
        fresh = (np.arange(nxt, nxt + a, dtype=np.uint64) * 2 + 1)
        nxt += a
        over = rng.integers(0, nxt, a).astype(np.uint64) * 2 + 1
        dele = rng.integers(0, 2 * nxt, n - 2 * a).astype(np.uint64)
        keys = np.concatenate([fresh, over, dele])
        ins = np.concatenate([np.ones(2 * a, np.uint8), np.zeros(n - 2 * a, np.uint8)])
        p = rng.permutation(n)
        keys, ins = keys[p], ins[p]
        yield [keys, rng.integers(0, 1 << 62, n).astype(np.uint64), rng.integers(0, 1 << 20, n).astype(np.uint64)], ins


def run_scale(be, ref, n_live=20_000_000, n=5_000_000, steps=5, seed=13):
    """A map of tens of millions of live keys, then `steps` steps of n mixed commands; every output bit for bit
    equal to the oracle's."""
    s = Schema("u", "uu")
    rng = np.random.default_rng(seed)
    runs = [Run(b, s, True) for b in (be, ref)]
    for t, (cols, ins) in enumerate(scale_steps(rng, n_live, n, steps)):
        for r in runs:
            r.h.append_columns(cols, ins)
            r.c.step()
        assert_batches_equal(runs[0].out.value, runs[1].out.value, f"scale step {t}")
        if t:
            assert len(runs[0].out.value) > n // 2, t
    return runs
