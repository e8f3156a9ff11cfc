#!/usr/bin/env python
"""The join probe (`join_delta_trace`: k_key_segments, k_probe_keys, k_row_counts_scan, k_probe_fill) at three shapes.

    python profiles/probe_bench.py [--calls 20] [--warmup 3]

Shapes (u64 key, u64 value; one row per trace key unless stated):
  * o1: q3's auctions against the person trace: ~10 M trace rows in 10 batches of halving size holding ascending key
    ranges (older batches hold older ids), 60 k delta rows whose keys fall in the newest batch;
  * o2: q3's persons against the auction trace: the same trace, 60 k delta rows above every trace key;
  * join: profiles/kernel_driver.py's join: 300 k random delta keys against 30 M random rows in 3 batches.  No batch
    can be skipped here: it isolates the shared search window.
Per shape: median, min and max ms of `calls` calls, each timed with CUDA events on the library's stream, the
matches per call, the trace's batch count, and the per-kernel profile of a second run of `calls` calls.  Prints one
JSON line per shape, with the card's name and power limit read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from rowfn_bench import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch

    from dbsp_b200 import Proj, Schema, Spine, key, lval, rval
    from dbsp_b200.runtime import Runtime

    be = Runtime(0)
    name, power = card()
    ext = torch.cuda.ExternalStream(be.stream_ptr, device=torch.device("cuda", 0))
    s = Schema("u", "u")
    proj = Proj(Schema("u", "uu"), [key(0), lval(0), rval(0)])
    rng = np.random.default_rng(0x9B0BE)

    def batch(keys):
        keys = np.sort(keys)
        return be.batch_from_columns(s, [keys, np.arange(len(keys), dtype=np.uint64)], np.ones(len(keys), np.int64))

    def spine(batches):
        sp = Spine(be, s)
        for k in batches:
            sp.insert(batch(k))
        return sp

    # ascending id ranges, halving sizes: 5 M, 2.5 M, ... (about 10 M rows), newest last
    sizes = [5_000_000 >> i for i in range(10)]
    starts = np.cumsum([0] + sizes)
    ids = spine([np.arange(starts[i], starts[i + 1], dtype=np.uint64) for i in range(10)])
    top = int(starts[-1])
    newest = (int(starts[-2]), top)
    rand = spine([rng.integers(0, 1 << 40, n, dtype=np.uint64) for n in (20_000_000, 7_000_000, 3_000_000)])
    shapes = {
        "o1": (ids, rng.integers(newest[0], newest[1], 60_000, dtype=np.uint64)),
        "o2": (ids, rng.integers(top, top + 60_000, 60_000, dtype=np.uint64)),
        "join": (rand, rng.integers(0, 1 << 40, 300_000, dtype=np.uint64)),
    }
    for label, (sp, dkeys) in shapes.items():
        d = batch(dkeys)
        for _ in range(args.warmup):
            out = be.join_delta_trace(d, sp, proj)
        matches = len(out)
        del out
        ms = []
        for _ in range(args.calls):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(ext)
            out = be.join_delta_trace(d, sp, proj)
            e1.record(ext)
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
            del out
        be.sync()
        be.profile(True)
        for _ in range(args.calls):
            be.join_delta_trace(d, sp, proj)
        be.sync()
        prof = be.profile_read()
        be.profile(False)
        print(json.dumps({"shape": label, "delta_rows": len(dkeys), "trace_rows": sp.stats()[0],
                          "trace_batches": sp.stats()[1], "matches_per_call": matches,
                          "median_ms": round(float(np.median(ms)), 4), "min_ms": round(min(ms), 4),
                          "max_ms": round(max(ms), 4),
                          "kernel_ms_per_call": {k: round(v["ms"] / args.calls, 4) for k, v in prof.items()},
                          "launches_per_call": {k: v["launches"] / args.calls for k, v in prof.items()},
                          "gpu": name, "power_limit_W_max_sm_MHz": power}), flush=True)


if __name__ == "__main__":
    main()
