#!/usr/bin/env python
"""Fold programs (dbsp_aggregate_fold) against the built-in aggregate kinds they equal, and Nexmark q6 / q18.

    python profiles/fold_bench.py [--rows 5000000] [--keys 1000000] [--hot 70000] [--reps 20] [--events 5000000]
                                  [--steps 6]

Inputs, each an OrdIndexedZSet<u64, u64> trace of one batch, aggregated for every key it holds (delta = the batch):
  * spread: `rows` rows over about `keys` keys;
  * hot: one key with `hot` rows, which one thread walks serially.
Per input, the median ms of `reps` calls (wall time between device syncs) of
  * fold_sum: Fold([0], [acc(0) + lval(0)]) against aggregate_delta(FOLD_SUM);
  * fold_max: Fold copying the last value against aggregate_delta(MAX).
The two results of each pair must be equal.  Then q6 and q18 on `steps` steps of `events` generated events: the
median ms of a step after the first (RootCircuit.step() between syncs).  Prints one JSON line per figure, with the
card's name and power limit read in the same run."""
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


def timed(be, fn, reps):
    out, ms = None, []
    for _ in range(reps + 1):
        be.sync()
        t0 = time.perf_counter()
        out = fn()
        be.sync()
        ms.append((time.perf_counter() - t0) * 1e3)
    return out, float(np.median(ms[1:]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=5_000_000)
    ap.add_argument("--keys", type=int, default=1_000_000)
    ap.add_argument("--hot", type=int, default=70_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--events", type=int, default=5_000_000)
    ap.add_argument("--steps", type=int, default=6)
    args = ap.parse_args()

    from dbsp_b200 import Fold, Proj, RootCircuit, Schema, Spine, acc, capi, lval
    from dbsp_b200.nexmark import NexmarkGenerator
    from dbsp_b200.nexmark import queries as nq
    from dbsp_b200.runtime import Runtime

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from parity_util import assert_batches_equal

    be = Runtime(0)
    name, power = card()
    s = Schema("u", "u")
    rng = np.random.default_rng(1)
    inputs = {
        "spread": [rng.integers(0, args.keys, args.rows).astype(np.uint64), rng.integers(0, 1 << 40, args.rows).astype(np.uint64)],
        "hot": [np.full(args.hot, 7, np.uint64), np.arange(args.hot, dtype=np.uint64) * np.uint64(3)],
    }
    folds = {"fold_sum": (Fold([0], [acc(0) + lval(0)]), capi.AGG_FOLD_SUM, Schema("u", "u")),
             "fold_max": (Fold([0], [lval(0)]), capi.AGG_MAX, s)}
    for inp, cols in inputs.items():
        b = be.batch_from_columns(s, cols)
        tr = Spine(be, s)
        tr.insert(b)
        for fname, (fold, kind, os_) in folds.items():
            ot = Spine(be, os_)
            got, ms_fold = timed(be, lambda: be.aggregate_fold(b, tr, ot, fold), args.reps)
            want, ms_kind = timed(be, lambda: be.aggregate_delta(b, tr, ot, kind), args.reps)
            assert_batches_equal(got, want, f"{fname} on {inp}")
            print(json.dumps({"input": inp, "rows": len(b), "keys": b.key_count(), "aggregate": fname,
                              "fold_ms": round(ms_fold, 3), "builtin_ms": round(ms_kind, 3), "card": name,
                              "power_limit_max_sm_clock": power}), flush=True)
    for q in ("q6", "q18"):
        gen = NexmarkGenerator(0x7FC359184519C0AA)
        c = RootCircuit(be)
        inp, handles = nq.add_nexmark_input(c)
        o = nq.QUERIES[q](inp).output()
        ms = []
        for st in range(args.steps):
            t = gen.tables(st * args.events, args.events)
            for k in ("person", "auction", "bid"):
                handles[k].set(t[k])
            be.sync()
            t0 = time.perf_counter()
            c.step()
            be.sync()
            ms.append((time.perf_counter() - t0) * 1e3)
        print(json.dumps({"query": q, "events_per_step": args.events, "steps": args.steps,
                          "median_step_ms": round(float(np.median(ms[1:])), 2), "last_output_rows": len(o.value),
                          "card": name, "power_limit_max_sm_clock": power}), flush=True)


if __name__ == "__main__":
    main()
