#!/usr/bin/env python
"""Fan-out against its host emulation, on Nexmark bids fanned out to their five HOP(2 s, 10 s) windows.

    python profiles/fanout_bench.py [--rows 5000000] [--reps 20] [--steps 5]

The closure is q5_hop's: (auction, starttime) for j = 0..4 with starttime = dt - dt % 2000 - 2000 * j, kept iff
2000 * j <= dt - dt % 2000.  Two inputs over one seeded 5 M-row bid sample, both already in HBM:
  * table: the raw bid columns.  dbsp_batch_from_table_fanout (n_out = 5) against five dbsp_batch_from_table_fn
    calls, one per j with j a constant, and four dbsp_batch_merge calls;
  * batch: the consolidated (auction, date_time) rows as a key-less batch.  dbsp_map_index_fanout against five
    dbsp_map_index_fn calls and four merges.
Each time is the median of `reps` runs, measured with CUDA events on the library's stream; it includes consolidation
and, for the emulation, the merges.  Both forms must give the same batch.  Then Nexmark q5_hop runs `steps` steps of
`rows` events from host tables; the per-step time is wall time around RootCircuit.step() and a device sync.  Prints
one JSON line per measurement with the card's name and power limit, read in the same run."""
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


def hop(schema, auction, dt, jv, n_out):
    """q5_hop's closure over the sources `auction` and `dt`: a fan-out for jv = fanout_index(), one run for a constant"""
    from dbsp_b200 import Proj
    from dbsp_b200.nexmark.queries import HOP_SLIDE_MS

    last = dt - dt.remu(HOP_SLIDE_MS)
    return Proj(schema, [auction, last - jv * HOP_SLIDE_MS], where=[(jv * HOP_SLIDE_MS).le(last)], fanout=n_out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=5_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()

    import torch

    from dbsp_b200 import RootCircuit, Schema, col, const, fanout_index, val
    from dbsp_b200.nexmark import NexmarkGenerator
    from dbsp_b200.nexmark import queries as nq
    from dbsp_b200.runtime import Runtime

    be = Runtime(0)
    name, power = card()
    gen = NexmarkGenerator(0x7FC359184519C0AA)
    n = args.rows
    bid = gen.tables(0, int(n / 0.92) + 1, want=("bid",))["bid"]   # 92 % of the events are bids
    cols = [torch.from_numpy(np.ascontiguousarray(c[:n]).view(np.int64)).cuda() for c in bid]
    n = int(cols[0].numel())
    ptrs = [c.data_ptr() for c in cols]
    k = nq.HOP_SIZE_MS // nq.HOP_SLIDE_MS
    pairs = be.batch_from_columns(Schema("", "uu"), [ptrs[0], ptrs[3]], n=n, on_device=True)   # (auction, date_time)

    s = Schema("uu")
    forms = {
        "table": (lambda: be.batch_from_table(ptrs, hop(s, col(0), col(3), fanout_index(), k), n=n, on_device=True),
                  [hop(s, col(0), col(3), const(jv), 1) for jv in range(k)],
                  lambda p: be.batch_from_table(ptrs, p, n=n, on_device=True)),
        "batch": (lambda: be.map_index(pairs, hop(s, val(0), val(1), fanout_index(), k)),
                  [hop(s, val(0), val(1), const(jv), 1) for jv in range(k)],
                  lambda p: be.map_index(pairs, p)),
    }
    stream = torch.cuda.ExternalStream(be.api._ctx_stream(be.ctx))

    def emulate(per_j, run):
        acc = run(per_j[0])
        for p in per_j[1:]:
            acc = be.merge(acc, run(p))
        return acc

    def timed(f):
        for _ in range(3):   # warm-up: module load, pool growth
            f()
        be.sync()
        times, rows = [], 0
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            out = f()
            b.record(stream)
            b.synchronize()
            times.append(a.elapsed_time(b))
            rows = len(out)
            del out
        return float(np.median(times)), float(np.min(times)), float(np.max(times)), rows

    for form, (fan, per_j, run) in forms.items():
        assert fan() == emulate(per_j, run), f"{form}: the fan-out and its emulation differ"
        for how, f in (("fanout", fan), ("emulation", lambda: emulate(per_j, run))):
            med, lo, hi, rows = timed(f)
            print(json.dumps({"input": form, "how": how, "rows": n, "n_out": k, "out_rows": rows, "median_ms": round(med, 3),
                              "min_ms": round(lo, 3), "max_ms": round(hi, 3), "gpu": name,
                              "power_limit_W_max_sm_MHz": power}), flush=True)
    del pairs

    # q5_hop per step: `rows` events per step from host tables
    c = RootCircuit(be)
    inp, handles = nq.add_nexmark_input(c)
    out = nq.QUERIES["q5_hop"](inp).output()
    times = []
    for step in range(args.steps + 1):
        t = gen.tables(step * args.rows, args.rows)
        for key_, h in handles.items():
            h.set(t[key_])
        be.sync()
        t0 = time.perf_counter()
        c.step()
        be.sync()
        if step:   # the first step is the warm-up
            times.append((time.perf_counter() - t0) * 1e3)
    print(json.dumps({"query": "q5_hop", "events_per_step": args.rows, "steps": args.steps,
                      "median_step_ms": round(float(np.median(times)), 2), "step_ms": [round(x, 2) for x in times],
                      "last_out_rows": len(out.value), "gpu": name, "power_limit_W_max_sm_MHz": power}), flush=True)


if __name__ == "__main__":
    main()
