#!/usr/bin/env python
"""Row functions against the fixed projection form on raw bid tables.

    python profiles/rowfn_bench.py [--rows 5000000] [--reps 20]

Times dbsp_batch_from_table (projection + filter + consolidation, columns already in HBM) with CUDA events on the
library's stream for four closures over one seeded 5 M-row bid table (columns auction, bidder, price, date_time,
extra): q4's bid projection `(auction, (price, date_time))` as a dbsp_proj and as the same closure compiled to a
dbsp_rowfn program, q1's `price * 89 / 100` and q2's `auction % 123 == 0` filter (programs only: neither fits a
dbsp_proj).  Prints one JSON line per closure: median ms, rows/s, and algorithmic GB/s = (the columns the closure
reads + the output rows and weights written by the projection) / time; the consolidation's own traffic is not
counted.  The card's name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=5_000_000)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()

    import torch

    from dbsp_b200 import Proj, Schema, col
    from dbsp_b200.nexmark import NexmarkGenerator
    from dbsp_b200.nexmark.queries import AUCTION_ID_MODULO
    from dbsp_b200.runtime import Runtime

    be = Runtime(0)
    gen = NexmarkGenerator(0x7FC359184519C0AA)
    n = args.rows
    bid = gen.tables(0, int(n / 0.92) + 1, want=("bid",))["bid"]   # 92 % of the events are bids
    cols = [torch.from_numpy(np.ascontiguousarray(c[:n]).view(np.int64)).cuda() for c in bid]
    n = int(cols[0].numel())
    ptrs = [c.data_ptr() for c in cols]

    q4 = Proj(Schema("u", "uu"), [col(0), col(2), col(3)])
    closures = {
        "q4_bid_proj": q4,
        "q4_bid_rowfn": q4.as_rowfn(),
        "q1_rowfn": Proj(Schema("uuuuu"), [col(0), col(1), (col(2) * 89).divu(100), col(3), col(4)]),
        "q2_rowfn": Proj(Schema("uu"), [col(0), col(2)], where=[col(0).remu(AUCTION_ID_MODULO).eq(0)]),
    }
    name, power = card()
    stream = torch.cuda.ExternalStream(be.api._ctx_stream(be.ctx))
    for label, p in closures.items():
        for _ in range(3):   # warm-up: module load, pool growth
            be.batch_from_table(ptrs, p, n=n, on_device=True)
        be.sync()
        times, out_rows = [], 0
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            out = be.batch_from_table(ptrs, p, n=n, on_device=True)
            b.record(stream)
            b.synchronize()
            times.append(a.elapsed_time(b))
            out_rows = len(out)
            del out
        ms = float(np.median(times))
        read = bin(be.proj_table_mask(p)).count("1") * 8 * n
        written = (p.schema.nl + 1) * 8 * out_rows
        print(json.dumps({"closure": label, "form": "dbsp_rowfn" if p.is_fn else "dbsp_proj", "rows": n,
                          "out_rows": out_rows, "median_ms": round(ms, 3), "rows_per_s": round(n / ms * 1e3),
                          "alg_GB_per_s": round((read + written) / ms / 1e6, 1), "gpu": name,
                          "power_limit_W_max_sm_MHz": power}), flush=True)


if __name__ == "__main__":
    main()
