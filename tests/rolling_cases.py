"""Partitioned rolling aggregates (dbsp_rolling_aggregate, Stream.partitioned_rolling_aggregate*) against a
non-incremental model: after every step, the integrated output equals the model over the integrated input, which
restates partitioned_rolling_aggregate_slow (operator/time_series/rolling_aggregate.rs:630-690).  Every case runs on a
list of backends; with two (the CUDA library and the CPU oracle) each step's output must also be bit-identical
between them.  ALL_CASES: name -> callable(*backends)."""
import bisect
import json
import os

import numpy as np

from dbsp_b200 import After, Before, Linear, Max, Min, Proj, RelRange, RootCircuit, Schema, Spine, key, lval, rval
from dbsp_b200._capi import DbspError

HERE = os.path.dirname(os.path.abspath(__file__))
M64 = (1 << 64) - 1


def _wrap(x, t):
    x &= M64
    return x - (1 << 64) if t == "i" and x >= 1 << 63 else x


# ---- the model -------------------------------------------------------------------------------------------------------
def model(integral: dict, schema: Schema, rng: RelRange, kind: str, f=None, f_types=""):
    """{(pk.., ts, some, agg..): 1} of the integral {(lanes..): weight} (lanes in natural form: i lanes signed).
    kind: 'max', 'min' or 'linear'; f(pk, v) -> (lanes, keep) with f_types the lanes' types.  Each window is
    aggregated on its own, over the partition's rows in ts order (numpy slices, wrapping u64 sums)."""
    nk, nvv = schema.nk, schema.nv - 1
    signed = schema.val[0] == "i"
    parts = {}
    for row, w in integral.items():
        if w != 0:
            parts.setdefault(row[:nk], []).append((row[nk], row[nk + 1:], w))
    n_agg = len(f_types) if kind == "linear" else nvv
    out = {}
    for pk, rows in parts.items():
        rows.sort()
        ts = [t for t, _, _ in rows]
        if kind == "linear":
            terms = []
            for _, v, w in rows:
                lanes, keep = f(pk, v)
                terms.append([(x * w) & M64 if keep else 0 for x in lanes])
            terms = np.array(terms, dtype=np.uint64).reshape(len(rows), n_agg)
        elif nvv == 1:
            vals = np.array([v[0] for _, v, _ in rows], dtype=np.int64 if schema.val[1] == "i" else np.uint64)
        for t in sorted({t for t, _, w in rows if w > 0}):
            r = rng.range_of(t, signed)
            if r is None:
                continue
            lo, hi = bisect.bisect_left(ts, r[0]), bisect.bisect_right(ts, r[1])
            if lo >= hi:
                out[pk + (t, 0) + (0,) * n_agg] = 1
                continue
            if kind == "linear":
                agg = tuple(_wrap(int(x), ty) for x, ty in zip(terms[lo:hi].sum(axis=0, dtype=np.uint64), f_types))
            elif nvv == 1:
                agg = (int(vals[lo:hi].max() if kind == "max" else vals[lo:hi].min()),)
            else:
                agg = (max if kind == "max" else min)(rows[j][1] for j in range(lo, hi))
            out[pk + (t, 1) + tuple(agg)] = 1
    return out


def _integrate(acc: dict, rows):
    for r in rows:
        acc[tuple(r[:-1])] = acc.get(tuple(r[:-1]), 0) + r[-1]
        if acc[tuple(r[:-1])] == 0:
            del acc[tuple(r[:-1])]


def _as_dict(rows):
    return {tuple(r[:-1]): r[-1] for r in rows}


# ---- the circuits ----------------------------------------------------------------------------------------------------
class Agg:
    """An aggregator and its model: 'max', 'min', or 'linear' with a Proj and its python twin."""

    def __init__(self, kind, proj=None, py=None):
        self.kind, self.proj, self.py = kind, proj, py

    def make(self):
        return {"max": Max, "min": Min}.get(self.kind) or Linear(self.proj)

    @property
    def f_types(self):
        return self.proj.schema.val if self.proj is not None else ""


def SUM0(vt="i"):
    """Linear sum of V lane 0 (the reference's Fold of val * w)"""
    return Agg("linear", Proj(Schema("", vt), [lval(0)]), lambda pk, v: ((v[0],), True))


COUNT = Agg("linear", Proj(Schema("", "i"), [1]), lambda pk, v: ((1,), True))


def build(be, schema: Schema, aggs, rng, lateness=None, comm=None):
    """One circuit: per aggregator, the plain form (lateness None) or the watermark form over the input re-indexed by
    its timestamp.  Returns (circuit, input handle, [(agg, output stream, integrated output node)])."""
    c = RootCircuit(be, comm)
    s, h = c.add_input_indexed_zset(schema)
    nk, nv = schema.nk, schema.nv
    outs = []
    if lateness is not None:
        by_ts = s.map_index(Proj(Schema(schema.val[0], schema.key + schema.val[1:]),
                                 [lval(0)] + [key(i) for i in range(nk)] + [lval(1 + j) for j in range(nv - 1)]))
        wm = by_ts.watermark_monotonic(lambda t: max(t - lateness, 0))
        part = Proj(Schema(schema.key, schema.val[1:]), [lval(i) for i in range(nk + nv - 1)])
    for a in aggs:
        if lateness is None:
            o = s.partitioned_rolling_aggregate(a.make(), rng)
        else:
            o = by_ts.partitioned_rolling_aggregate_with_watermark(wm, part, a.make(), rng)
        integ = o.gather(0).integrate() if comm is not None else o.integrate()
        outs.append((a, o, integ.output(), o.output()))
    return c, h, outs


def check_bounds(o, cap=None):
    """The watermark form's state: every row of the operator's input and output traces (consolidated, which applies
    the output trace's bound) and of its window has ts >= the current lower bound; with `cap`, each of the three
    traces also physically holds at most `cap` rows (spine_len, every batch's rows before consolidation), the
    counterpart of the reference's size bound on the output trace."""
    lower = o.rolling_lower()
    for tr, col in ((o.rolling_in_trace, o.rolling_in_trace.schema.nk), (o.rolling_out_trace, o.rolling_out_trace.schema.nk),
                    (o.window_trace, 0)):
        signed = tr.schema.lanes[col] == "i"
        for r in tr.consolidate().rows():
            assert r[col] >= (lower if not signed or lower < 1 << 63 else lower - (1 << 64)), (r, lower)
        if cap is not None:
            assert tr.stats()[0] <= cap, (tr.schema, tr.stats(), cap)


def run(bes, schema: Schema, steps, rng, aggs, lateness=None, cap=None, after_step=None):
    """Feed `steps` (lists of (lanes.., weight) rows) to one circuit per backend; after every step compare each
    integrated output with the model, and the step's outputs across the backends.  cap: see check_bounds;
    after_step(i, outs) runs after step i on each backend's outputs."""
    runs = [build(be, schema, aggs, rng, lateness) for be in bes]
    integral = {}
    for i, rows in enumerate(steps):
        for c, h, _ in runs:
            h.append(rows)
            c.step()
        _integrate(integral, rows)
        wants = [model(integral, schema, rng, a.kind, a.py, a.f_types) for a in aggs]
        deltas = []
        for c, h, outs in runs:
            ds = []
            for want, (a, o, integ, delta) in zip(wants, outs):
                got = _as_dict(integ.value.rows())
                assert got == want, f"step {i} {a.kind} {rng}: {sorted(set(got.items()) ^ set(want.items()))[:6]}"
                if lateness is not None:
                    check_bounds(o, cap)
                ds.append(delta.value.rows())
            if after_step is not None:
                after_step(i, outs)
            deltas.append(ds)
        for d in deltas[1:]:
            assert d == deltas[0], f"step {i}: the backends' outputs differ"


# ---- the cases -------------------------------------------------------------------------------------------------------
REF_RANGES = [RelRange(Before(1000), Before(0)), RelRange(Before(500), After(500)), RelRange(Before(500), Before(100))]
REF_SCHEMA = Schema("u", "ui")
REF_AGGS = [SUM0(), Agg("max"), Agg("min")]
# The quasi-monotone strategy adds up to 20 rows per step to a window of 10 000 that moves by 2 000; with the watermark
# 10 000 behind the newest time and the ranges at most 1 000 wide, a step's live input spans about 11 steps of rows
# (~220; each trace held at most 116 in the seeded run).  Unbounded, they would grow to the 200 steps' ~2 000 rows.
QUASI_CAP = 300


def _golden(name):
    with open(os.path.join(HERE, "golden", "rolling_aggregate.json")) as fh:
        return json.load(fh)[name]


def _reference(name, lateness):
    def case(*bes):
        for rng in REF_RANGES:
            run(bes, REF_SCHEMA, _golden(name), rng, REF_AGGS, lateness)
    return case


def _proptest(seed, parts, epoch, max_rows, n_steps, lateness=None, quasi=None, cap=None):
    """Seeded versions of the reference's strategies: rows (p < parts, ts in the step's window, 100, +1).  cap: the
    watermark form's bound on each trace's physical rows (check_bounds)."""
    def case(*bes):
        r = np.random.default_rng(seed)
        steps = []
        for i in range(n_steps):
            lo, hi = (i * quasi[1], i * quasi[1] + quasi[0]) if quasi else (0, epoch)
            n = int(r.integers(0, max_rows))
            steps.append([(int(p), int(t), 100, 1) for p, t in zip(r.integers(0, parts, n), r.integers(lo, hi, n))])
        for rng in REF_RANGES:
            run(bes, REF_SCHEMA, steps, rng, REF_AGGS)
            run(bes, REF_SCHEMA, steps, rng, REF_AGGS, M64 >> 1 if lateness is None else lateness, cap)
    return case


def case_retract_last_positive(*bes):
    steps = [[(0, 10, 5, 1), (0, 20, 7, 1), (0, 20, 8, 1)], [(0, 20, 7, -1)], [(0, 20, 8, -1)], [(0, 10, 5, -1)]]
    for rng in REF_RANGES[:2]:
        run(bes, REF_SCHEMA, steps, rng, REF_AGGS)


def case_negative_only(*bes):
    """a ts whose only row has negative weight gets no output, yet its row is in the neighbours' windows"""
    steps = [[(0, 10, 5, -1), (0, 12, 9, 1)], [(0, 11, 3, -2), (0, 10, 6, 1)], [(0, 10, 6, -1)]]
    run(bes, REF_SCHEMA, steps, RelRange(Before(5), After(5)), REF_AGGS)


def case_weights_wrapping(*bes):
    big = (1 << 62) + 7
    steps = [[(1, 3, big, 3), (1, 4, -big, 5), (1, 5, 11, -4)], [(1, 6, big, 7), (1, 4, -big, -5)]]
    run(bes, REF_SCHEMA, steps, RelRange(Before(2), After(1)), [SUM0(), COUNT, Agg("max")])


def case_insert_delete_batches(*bes):
    """a row inserted and deleted in different trace batches before they merge (the trace holds +1 and -1)"""
    steps = [[(0, 5, 1, 1)] + [(0, 100 + i, i, 1) for i in range(40)], [(0, 7, 2, 1)], [(0, 5, 1, -1)], [(0, 6, 3, 1)]]
    run(bes, REF_SCHEMA, steps, RelRange(Before(3), Before(0)), REF_AGGS)


def case_ranges_excluding_ts(*bes):
    """After..After and Before..Before ranges that exclude ts (some = 0), and zero-width ranges"""
    steps = [[(0, 1, 4, 1), (0, 3, 9, 1), (1, 10, 2, 1)], [(0, 2, 1, 1), (1, 11, 5, 1)], [(0, 3, 9, -1)]]
    for rng in (RelRange(After(1), After(1)), RelRange(After(1), After(5)), RelRange(Before(2), Before(1)),
                RelRange(Before(0), Before(0)), RelRange(After(0), After(0)), RelRange(Before(0), After(0))):
        run(bes, REF_SCHEMA, steps, rng, REF_AGGS)


def case_range_limits_u64(*bes):
    """range_of = None near 0 (a `to` Before underflows) and near 2^64 (a `from` After overflows)"""
    top = M64
    steps = [[(0, 0, 1, 1), (0, 3, 2, 1), (0, top, 5, 1), (0, top - 2, 6, 1)], [(0, 1, 7, 1), (0, top - 1, 3, 1)]]
    for rng in (RelRange(Before(2), Before(2)), RelRange(After(2), After(3)), RelRange(Before(top), After(top)),
                RelRange(Before(5), After(top))):
        run(bes, REF_SCHEMA, steps, rng, REF_AGGS)


def case_range_limits_i64(*bes):
    """i64 timestamps below 0 and at both ends of i64"""
    lo, hi = -(1 << 63), (1 << 63) - 1
    s = Schema("u", "ii")
    steps = [[(0, -5, 1, 1), (0, -1, 2, 1), (0, lo, 3, 1), (0, hi, 4, 1)], [(0, lo + 1, -7, 1), (0, 0, 5, 1), (0, hi - 1, 8, 1)]]
    for rng in (RelRange(Before(3), After(1)), RelRange(After(1), After(2)), RelRange(Before(2), Before(1)),
                RelRange(Before(hi), After(hi))):
        run(bes, s, steps, rng, [SUM0(), Agg("max"), Agg("min")])


def case_wide_keys(*bes):
    """3-lane (signed) partition keys, and key-less ones (one partition)"""
    r = np.random.default_rng(5)
    s3 = Schema("uiu", "ui")
    steps3 = [[(int(a), int(b), int(c), int(t), int(v), int(w)) for a, b, c, t, v, w in
               zip(r.integers(0, 2, 30), r.integers(-2, 2, 30), r.integers(0, 2, 30), r.integers(0, 40, 30),
                   r.integers(-9, 9, 30), r.choice([-1, 1, 2], 30))] for _ in range(5)]
    run(bes, s3, steps3, RelRange(Before(5), After(2)), REF_AGGS)
    s0 = Schema("", "ui")
    steps0 = [[(int(t), int(v), int(w)) for t, v, w in zip(r.integers(0, 60, 25), r.integers(-9, 9, 25), r.choice([-1, 1], 25))]
              for _ in range(5)]
    run(bes, s0, steps0, RelRange(Before(7), Before(0)), REF_AGGS)


def case_two_lane_values(*bes):
    """Max / Min over 2-lane i64 values, and a 3-lane Linear f with a keep flag"""
    r = np.random.default_rng(8)
    s = Schema("u", "uii")
    steps = [[(int(p), int(t), int(a), int(b), 1) for p, t, a, b in
              zip(r.integers(0, 3, 40), r.integers(0, 50, 40), r.integers(-3, 3, 40), r.integers(-1 << 62, 1 << 62, 40))]
             for _ in range(5)]
    f = Agg("linear", Proj(Schema("", "iui"), [lval(0) * 3, lval(1), key(0) + lval(0)], [lval(0).ge(0).signed()]),
            lambda pk, v: ((v[0] * 3, v[1], pk[0] + v[0]), v[0] >= 0))
    run(bes, s, steps, RelRange(Before(10), After(3)), [Agg("max"), Agg("min"), f])


def case_many_batches(*bes):
    """a trace of 18 batches, more than one gather chunk (MAX_REFS = 16): step i inserts 2^(17-i) new rows, so no two
    batches of the input trace merge, and each step's window (the whole partition) reads every batch"""
    r = np.random.default_rng(17)
    steps, v = [], 0
    for i in range(18):
        n = 1 << (17 - i)
        steps.append([(int(p), int(t), v + j, 1) for j, (p, t) in enumerate(zip(r.integers(0, 2, n), r.integers(0, 1000, n)))])
        v += n

    def batches(i, outs):
        for _, o, _, _ in outs:
            assert o.rolling_in_trace.stats()[1] == i + 1, (i, o.rolling_in_trace.stats())

    run(bes, REF_SCHEMA, steps, RelRange(Before(1000), After(1000)), REF_AGGS, after_step=batches)


def case_hot_window(*bes):
    """one partition with 70 000 rows in one window (the sparse table and the prefix sums over many blocks)"""
    r = np.random.default_rng(3)
    n = 70_000
    ts, v = r.integers(0, 1000, n), r.integers(-1 << 40, 1 << 40, n)
    s1 = [(0, int(t), int(x), 1) for t, x in zip(ts, v)]
    s2 = [(0, int(t), int(x), -1) for t, x in zip(ts[:500], v[:500])] + [(0, 500, 1 << 41, 1)]
    run(bes, REF_SCHEMA, [s1, s2], RelRange(Before(1000), Before(0)), REF_AGGS)


def case_empty_steps(*bes):
    run(bes, REF_SCHEMA, [[], [(0, 3, 1, 1)], [], [], [(0, 3, 1, -1)], []], RelRange(Before(2), After(2)), REF_AGGS)


# ---- Nexmark rolling_bids -------------------------------------------------------------------------------------------
BID_SCHEMA = Schema("u", "uu")   # auction -> (date_time, price)
BID_AGGS = [Agg("linear", Proj(Schema("", "ii"), [1, lval(0)]), lambda pk, v: ((1, v[0]), True)), Agg("max")]


def _bids_circuit(be, watermark):
    from dbsp_b200.nexmark import queries as nq

    c = RootCircuit(be)
    inp, handles = nq.add_nexmark_input(c)
    return c, handles, nq.rolling_bids(inp, watermark)


def run_bids_model(be, watermark, n_events=2_000, steps=10):
    """rolling_bids on generated events (2 000 events per second of event time, so that a one-second window holds a
    few bids of an auction, and a step spans one second, well within the watermark's lateness): after every step both
    integrated outputs equal the model over the bids so far"""
    from dbsp_b200.nexmark import NexmarkGenerator
    from dbsp_b200.nexmark import queries as nq

    gen = NexmarkGenerator(0x7FC359184519C0AA, first_event_rate=2_000)
    c, handles, outs = _bids_circuit(be, watermark)
    integ = [o.integrate().output() for o in outs]
    bids = {}
    for s in range(steps):
        t = gen.tables(s * n_events, n_events)
        for k in ("person", "auction", "bid"):
            handles[k].set(t[k])
        c.step()
        _integrate(bids, [(a, ts, p, 1) for a, _, p, ts, _ in zip(*[x.tolist() for x in t["bid"]])])
        for a, node in zip(BID_AGGS, integ):
            want = model(bids, BID_SCHEMA, nq.ROLLING_RANGE, a.kind, a.py, a.f_types)
            got = _as_dict(node.value.rows())
            assert got == want, (s, a.kind, watermark, len(got), len(want))
            if a.kind == "linear":
                counts = [r[3] for r in want]
    assert len(bids) > 10_000 and max(counts) > 1   # windows that hold several bids of an auction


def run_bids_pair(be, ref, watermark, n_events=5_000_000, steps=5):
    """rolling_bids at the default event rate: every step's two outputs bit-identical between `be` and `ref`"""
    from dbsp_b200.nexmark import NexmarkGenerator

    gen = NexmarkGenerator(0x7FC359184519C0AA)
    runs = [_bids_circuit(b, watermark) for b in (be, ref)]
    for s in range(steps):
        t = gen.tables(s * n_events, n_events)
        got = []
        for c, handles, outs in runs:
            for k in ("person", "auction", "bid"):
                handles[k].set(t[k])
            c.step()
            got.append([o.node.value.download() for o in outs])
        for x, y in zip(*got):
            for k in ("keys", "vals"):
                for a, b in zip(x[k], y[k]):
                    assert np.array_equal(np.asarray(a), np.asarray(b)), (s, k, watermark)
            assert np.array_equal(x["offs"], y["offs"]) and np.array_equal(x["diffs"], y["diffs"]), (s, watermark)
            assert len(x["diffs"]) > 0


ALL_CASES = {
    "reference_over_range": _reference("test_partitioned_over_range", None),
    "reference_over_range_2": _reference("test_partitioned_over_range_2", None),
    "reference_over_range_watermark": _reference("test_partitioned_over_range", M64 >> 1),
    "reference_over_range_2_watermark": _reference("test_partitioned_over_range_2", M64 >> 1),
    "proptest_dense": _proptest(11, 5, 1_000, 50, 20),
    "proptest_sparse": _proptest(12, 5, 1_000_000, 20, 20),
    "proptest_quasi_monotone": _proptest(13, 5, None, 20, 200, lateness=10_000, quasi=(10_000, 2_000), cap=QUASI_CAP),
    "retract_last_positive": case_retract_last_positive,
    "negative_only": case_negative_only,
    "weights_wrapping": case_weights_wrapping,
    "insert_delete_batches": case_insert_delete_batches,
    "ranges_excluding_ts": case_ranges_excluding_ts,
    "range_limits_u64": case_range_limits_u64,
    "range_limits_i64": case_range_limits_i64,
    "wide_keys": case_wide_keys,
    "two_lane_values": case_two_lane_values,
    "many_batches": case_many_batches,
    "hot_window": case_hot_window,
    "empty_steps": case_empty_steps,
    "rolling_bids": lambda *bes: [run_bids_model(be, False) for be in bes],
    "rolling_bids_watermark": lambda *bes: [run_bids_model(be, True) for be in bes],
}


# ---- refusals --------------------------------------------------------------------------------------------------------
def refusals(be):
    """One call per rule of validate.h's valid_rolling: [(rule, status, text)]."""
    s = REF_SCHEMA
    d = be.batch_from_rows(s, [(0, 1, 1, 1)])
    it = Spine(be, s)
    lin_out = Spine(be, Schema("u", "uui"))
    mm_out = Spine(be, Schema("u", "uui"))
    ok = RelRange(Before(1), Before(0))
    f = Proj(Schema("", "i"), [lval(0)])
    out = []

    def call(rule, *args):
        try:
            be.rolling_aggregate(*args)
        except DbspError as e:
            out.append((rule, str(e)))
            return
        raise AssertionError(f"{rule}: accepted")

    ts_only = Schema("u", "u")
    call("delta and in_trace differ", d, Spine(be, Schema("u", "uu")), lin_out, ok, 0, f)
    call("no value lane", be.batch_from_rows(Schema("u"), [(0, 1)]), Spine(be, Schema("u")), lin_out, ok, 0, f)
    call("max without V", be.batch_from_rows(ts_only, [(0, 1, 1)]), Spine(be, ts_only), Spine(be, Schema("u", "uu")), ok, 1)
    call("kind outside the enum", d, it, mm_out, ok, 3)
    call("LINEAR without f", d, it, lin_out, ok, 0)
    call("f for MAX", d, it, mm_out, ok, 1, f)
    wide = Schema("uuuuu", "uuu")   # PK 5 + ts + some + 2 V lanes = 9
    call("MAX too wide", be.batch_from_rows(wide, [(0,) * 8 + (1,)]), Spine(be, wide), Spine(be, Schema("uuuuu", "uuu")), ok, 1)
    call("f with key lanes", d, it, lin_out, ok, 0, Proj(Schema("i"), [lval(0)]))
    call("f too wide", d, it, lin_out, ok, 0, Proj(Schema("", "iiiiii"), [lval(0)] * 6))
    call("f reads RVAL", d, it, lin_out, ok, 0, Proj(Schema("", "i"), [lval(0) + rval(0)]).as_rowfn())
    call("out_trace schema", d, it, Spine(be, Schema("u", "uii")), ok, 0, f)
    call("reversed range", d, it, lin_out, RelRange(Before(0), Before(1)), 0, f)
    call("reversed After..Before", d, it, lin_out, RelRange(After(1), Before(0)), 0, f)
    si = Schema("u", "ii")
    call("i64 offset", be.batch_from_rows(si, [(0, 1, 1, 1)]), Spine(be, si), Spine(be, Schema("u", "iui")),
         RelRange(Before(1 << 63), Before(0)), 1)
    return out


def run_refusals(be):
    got = refusals(be)
    assert len(got) == 14
    for rule, text in got:
        assert "rolling_aggregate" in text and "INVALID" in text, (rule, text)
    return [(rule, text.split(" failed: ", 1)[1]) for rule, text in got]
