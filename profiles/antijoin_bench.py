#!/usr/bin/env python
"""Stream.antijoin and Stream.outer_join against the reference's compositions, step by step.

    python profiles/antijoin_bench.py [--rows 5000000] [--keys 1000000] [--steps 20] [--warmup 2]

Both sides start with `rows` rows (u64 key, u64 value) over about `keys` keys, loaded in one step that is not timed.
Three inputs follow, each for warmup + steps steps on both sides:
  * 1 % and 10 %: deltas of rows/100 and rows/10 rows, a quarter of them retractions of loaded rows;
  * skew: 1 % deltas, where every delta also adds 100 rows on the hot key.
The hot key gets 10 000 rows on each side in a second untimed step after the load, so all three inputs run with it
in the traces; only the skew deltas touch it.
Four circuits get the same inputs, alternating within each step:
  * antijoin: Stream.antijoin (dbsp_antijoin_delta);
  * antijoin_composed: self − self ⋈ distinct(other), built here from join, distinct and minus (join.rs:294-320);
  * outer_join: Stream.outer_join with fl / fr = f with the other side's value read as 0;
  * outer_join_composed: join(f) + composed antijoin(a, b).map(fl) + composed antijoin(b, a).map(fr) (join.rs:332-360).
Each new circuit's output must equal its composition's at every step.  Per circuit and input: the median ms of a step
(wall time around RootCircuit.step() between device syncs), kernel launches and host read-backs per step, and the
rows its spines hold after the last step.  Prints one JSON line each, with the card's name and power limit read in
the same run."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from rowfn_bench import card  # noqa: E402

HOT, HOT_ROWS, HOT_DELTA = 1 << 40, 10_000, 100


def spine_rows(circuit):
    """Rows held by the spines the circuit's operators own (found in their closures)."""
    from dbsp_b200.circuit import _KeyCounts
    from dbsp_b200.zset import Spine

    seen, rows = set(), 0
    for n in circuit.nodes:
        for cell in n.fn.__closure__ or ():
            v = cell.cell_contents
            sp = v.trace if isinstance(v, _KeyCounts) else v
            if isinstance(sp, Spine) and id(sp) not in seen:
                seen.add(id(sp))
                rows += sp.stats()[0]
    return rows


def composed_antijoin(a, b, s):
    from dbsp_b200 import Proj, key, lval

    ident = Proj(s, [key(0), lval(0)])
    return a.minus(a.join(b.distinct(), ident))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=5_000_000)
    ap.add_argument("--keys", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    from dbsp_b200 import Proj, RootCircuit, Schema, const, key, lval, rval
    from dbsp_b200.runtime import Runtime

    be = Runtime(0)
    name, power = card()
    s, so = Schema("u", "u"), Schema("u", "uu")
    f = Proj(so, [key(0), lval(0), rval(0)])
    fl, fr = Proj(so, [key(0), lval(0), const(0)]), Proj(so, [key(0), const(0), rval(0)])
    rng = np.random.default_rng(0x5EED)

    def rows(n, keys=None):
        k = rng.integers(0, args.keys, n, dtype=np.uint64) if keys is None else keys
        return [k, rng.integers(0, 1 << 40, n, dtype=np.uint64)], np.ones(n, np.int64)

    base = [rows(args.rows), rows(args.rows)]

    def delta(n, side, skew):
        (k, v), w = rows(n - n // 4)
        pick = rng.integers(0, args.rows, n // 4)   # retract loaded rows
        k = np.concatenate([k, base[side][0][0][pick]])
        v = np.concatenate([v, base[side][0][1][pick]])
        w = np.concatenate([w, -np.ones(n // 4, np.int64)])
        if skew:
            k[:HOT_DELTA] = HOT
        return [k, v], w

    circuits = {}
    for kind in ("antijoin", "antijoin_composed", "outer_join", "outer_join_composed"):
        c = RootCircuit(be)
        st = {}
        a = c.add_source(lambda st=st: st["a"], s)
        b = c.add_source(lambda st=st: st["b"], s)
        if kind == "antijoin":
            o = a.antijoin(b)
        elif kind == "antijoin_composed":
            o = composed_antijoin(a, b, s)
        elif kind == "outer_join":
            o = a.outer_join(b, f, fl, fr)
        else:
            o = a.join(b, f).sum([composed_antijoin(a, b, s).map(fl), composed_antijoin(b, a, s).map(fr)])
        circuits[kind] = (c, st, o.output())

    def step(inputs):
        """One step of every circuit on the same host inputs; returns {kind: (ms, launches, read-backs)}."""
        res = {}
        for kind, (c, st, _) in circuits.items():
            st["a"] = be.batch_from_columns(s, *inputs[0])
            st["b"] = be.batch_from_columns(s, *inputs[1])
            be.sync()
            be.stats(reset=True)
            t0 = time.perf_counter()
            c.step()
            be.sync()
            ms = (time.perf_counter() - t0) * 1e3
            x = be.stats(reset=True)
            res[kind] = (ms, x["kernel_launches"], x["host_waits"])
        for new in ("antijoin", "outer_join"):
            assert circuits[new][2].value == circuits[new + "_composed"][2].value, f"{new} differs from its composition"
        return res

    step(base)   # the load step
    hot = [(([np.full(HOT_ROWS, HOT, np.uint64), np.arange(HOT_ROWS, dtype=np.uint64) * np.uint64(side + 1)],
             np.ones(HOT_ROWS, np.int64))) for side in (0, 1)]
    step(hot)
    for label, frac, skew in (("1%", 0.01, False), ("10%", 0.10, False), ("skew", 0.01, True)):
        n = int(args.rows * frac)
        got = {k: [] for k in circuits}
        for t in range(args.warmup + args.steps):
            r = step([delta(n, 0, skew), delta(n, 1, skew)])
            if t >= args.warmup:
                for k, v in r.items():
                    got[k].append(v)
        for kind, v in got.items():
            ms = [x[0] for x in v]
            print(json.dumps({"input": label, "circuit": kind, "rows_per_side": args.rows, "keys": args.keys,
                              "delta_rows_per_side": n, "median_step_ms": round(float(np.median(ms)), 3),
                              "min_ms": round(min(ms), 3), "max_ms": round(max(ms), 3),
                              "launches_per_step": float(np.median([x[1] for x in v])),
                              "readbacks_per_step": float(np.median([x[2] for x in v])),
                              "spine_rows": spine_rows(circuits[kind][0]), "gpu": name,
                              "power_limit_W_max_sm_MHz": power}), flush=True)


if __name__ == "__main__":
    main()
