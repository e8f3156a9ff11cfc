#!/usr/bin/env python
"""Nexmark `rolling_bids` (count, sum and max price of each auction's bids over the last second), per step, on the GPU
and on the CPU oracle, in its plain and watermark forms.

    python profiles/rolling_bench.py [--events 5000000] [--steps 5] [--oracle-steps 2] [--backend both|cuda|oracle]

Each step feeds `events` generated Nexmark events (default event rate) to one circuit with both aggregates of one
form, with a device sync after the step.  The median of the steps after the first is printed per backend and form.
On the GPU a further profiled step splits the time by kernel class: `rolling` (the affected intervals, the range
gather's search and copy, the prefix-sum terms, the sparse table, the outputs, the retractions), `merge_tiles` (the
merge tree of the gathered slices and of old and new outputs), `radix_sort` / `heads` / `emit` (the consolidation of
the intervals and of the bid projection), `scan`, and the rest.  One JSON line per figure, with the card's name and
power limit read in the same run (`--backend oracle` needs no GPU and records none)."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))


def circuit(be, watermark):
    from dbsp_b200 import RootCircuit
    from dbsp_b200.nexmark import queries as nq

    c = RootCircuit(be)
    inp, handles = nq.add_nexmark_input(c)
    outs = [o.output() for o in nq.rolling_bids(inp, watermark)]
    return c, handles, outs


def run(be, watermark, steps, prof):
    """Per-step ms, the last step's output rows, and (prof) the kernel classes of one more profiled step."""
    from dbsp_b200.nexmark import NexmarkGenerator

    gen = NexmarkGenerator(0x7FC359184519C0AA)
    c, handles, outs = circuit(be, watermark)

    def feed(s):
        t = gen.tables(s * args.events, args.events)
        for k in ("person", "auction", "bid"):
            handles[k].set(t[k])

    ms, rows = [], 0
    for s in range(steps):
        feed(s)
        be.sync()
        t0 = time.perf_counter()
        c.step()
        be.sync()
        ms.append((time.perf_counter() - t0) * 1e3)
        rows = sum(len(o.value) for o in outs)
    classes = None
    if prof:
        feed(steps)
        be.sync()
        be.profile(True)
        c.step()
        be.sync()
        classes = {k: {"ms": round(v["ms"], 3), "launches": v["launches"], "alg_MB": round(v["alg_bytes"] / 1e6, 1)}
                   for k, v in be.profile_read().items()}
        be.profile(False)
    return ms, rows, classes


def main():
    from rowfn_cases import fn_oracle

    name = power = None
    if args.backend in ("both", "cuda"):
        from dbsp_b200.runtime import Runtime
        from rowfn_bench import card

        name, power = card()
        cuda = Runtime(0)
        for wm in (False, True):
            ms, rows, classes = run(cuda, wm, args.steps, prof=True)
            print(json.dumps({"backend": "cuda", "form": "watermark" if wm else "plain", "events": args.events,
                              "steps": args.steps, "step_ms": round(float(np.median(ms[1:] or ms)), 2),
                              "out_rows": rows, "kernel_classes": classes, "card": name,
                              "power_limit_max_sm_clock": power}), flush=True)
    if args.backend in ("both", "oracle"):
        orc = fn_oracle()
        for wm in (False, True):
            ms, rows, _ = run(orc, wm, args.oracle_steps, prof=False)
            print(json.dumps({"backend": "oracle", "form": "watermark" if wm else "plain", "events": args.events,
                              "steps": args.oracle_steps, "step_ms": round(float(np.median(ms[1:] or ms)), 1),
                              "out_rows": rows, "card": name, "power_limit_max_sm_clock": power}), flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--events", type=int, default=5_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--oracle-steps", type=int, default=2)
    ap.add_argument("--backend", choices=("both", "cuda", "oracle"), default="both")
    args = ap.parse_args()
    main()
