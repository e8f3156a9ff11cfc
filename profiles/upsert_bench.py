#!/usr/bin/env python
"""One step of a map input table (dbsp_upsert_commands + dbsp_upsert_delta + the trace insert), by stage, on the GPU
and on the CPU oracle.

    python profiles/upsert_bench.py [--live 50000000] [--cmds 5000000] [--steps 5] [--oracle-steps 2]

The table is an OrdIndexedZSet<u64, (u64, u64)> map of `live` keys, loaded into its trace as one batch.  Each step
applies `cmds` commands, shuffled: a third inserts of fresh keys, a third overwrites of live keys, a third deletes
(half of them of absent keys).  Per step, with a device sync around each stage:
  * commands: dbsp_upsert_commands over resident device columns (the command build and its consolidation sort);
  * delta: dbsp_upsert_delta (last command per key, the probe of the table's trace, negate, merge);
  * insert: the insert of the delta into the table's trace (the spine's merges it triggers).
`step_ms` is the three without syncs between them.  The medians of the steps after the first are printed, and, from a
separate profiled step, the kernel classes of the delta: `upsert` (k_upsert_last), `probe_ranges` / `probe_fill`
(the trace probe), `merge_tiles` (the merge of the new rows with the retractions).  Then the same steps on the CPU
oracle over the same table.  One JSON line per figure, with the card's name and power limit read in the same run."""
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

from rowfn_bench import card  # noqa: E402


def step_commands(rng, n_live, n, t):
    a = n // 3
    fresh = np.arange(n_live + t * a, n_live + (t + 1) * a, dtype=np.uint64) * np.uint64(2)
    over = rng.integers(0, n_live, a).astype(np.uint64) * np.uint64(2)
    dele = rng.integers(0, 2 * n_live, n - 2 * a).astype(np.uint64)
    keys = np.concatenate([fresh, over, dele])
    ins = np.concatenate([np.ones(2 * a, np.uint8), np.zeros(n - 2 * a, np.uint8)])
    p = rng.permutation(n)
    return [keys[p], rng.integers(0, 1 << 62, n).astype(np.uint64), rng.integers(0, 1 << 20, n).astype(np.uint64)], ins[p]


def run(be, s, table, steps, device, prof=False):
    """Per step (stage ms..., step ms) and the last step's delta."""
    import torch

    rng = np.random.default_rng(5)
    out, rows, classes = [], None, None
    for t in range(steps):
        cols, ins = step_commands(rng, args.live, args.cmds, t)
        if device:
            dc = [torch.from_numpy(c.view(np.int64)).cuda() for c in cols]
            di = torch.from_numpy(ins).cuda()
            mk = lambda: be.upsert_commands(s, [int(c.data_ptr()) for c in dc], int(di.data_ptr()), n=len(ins), on_device=True)  # noqa: E731
        else:
            mk = lambda: be.upsert_commands(s, cols, ins)  # noqa: E731
        be.sync()
        t0 = time.perf_counter()
        cmds = mk()
        be.sync()
        t1 = time.perf_counter()
        d = be.upsert_delta(cmds, table)
        be.sync()
        t2 = time.perf_counter()
        table.insert(d)
        be.sync()
        t3 = time.perf_counter()
        out.append(((t1 - t0) * 1e3, (t2 - t1) * 1e3, (t3 - t2) * 1e3))
        rows = len(d)
    if prof:
        cols, ins = step_commands(rng, args.live, args.cmds, steps)
        cmds = be.upsert_commands(s, cols, ins)
        be.sync()
        be.profile(True)
        table.insert(be.upsert_delta(cmds, table))
        classes = {k: round(v["ms"], 3) for k, v in be.profile_read().items()}
        be.profile(False)
    return out, rows, classes


def whole_steps(be, s, table, steps):
    import torch

    rng = np.random.default_rng(6)
    ms = []
    for t in range(steps):
        cols, ins = step_commands(rng, args.live, args.cmds, 100 + t)
        dc = [torch.from_numpy(c.view(np.int64)).cuda() for c in cols]
        di = torch.from_numpy(ins).cuda()
        be.sync()
        t0 = time.perf_counter()
        cmds = be.upsert_commands(s, [int(c.data_ptr()) for c in dc], int(di.data_ptr()), n=len(ins), on_device=True)
        table.insert(be.upsert_delta(cmds, table))
        be.sync()
        ms.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ms[1:]))


def load(be, s):
    from dbsp_b200 import Spine

    k = np.arange(args.live, dtype=np.uint64) * np.uint64(2)
    tr = Spine(be, s)
    tr.insert(be.batch_from_columns(s, [k, k * np.uint64(7), k & np.uint64(1023)]))
    return tr


def main():
    from dbsp_b200 import Schema
    from dbsp_b200.runtime import Runtime
    from rowfn_cases import fn_oracle

    name, power = card()
    s = Schema("u", "uu")
    be = Runtime(0)
    table = load(be, s)
    per, rows, classes = run(be, s, table, args.steps, device=True, prof=True)
    med = np.median(np.array(per[1:]), axis=0)
    print(json.dumps({"backend": "cuda", "live_keys": args.live, "commands": args.cmds, "steps": args.steps,
                      "commands_ms": round(med[0], 2), "delta_ms": round(med[1], 2), "insert_ms": round(med[2], 2),
                      "step_ms": round(whole_steps(be, s, table, args.steps), 2), "delta_rows": rows,
                      "delta_kernel_ms": classes, "card": name, "power_limit_max_sm_clock": power}), flush=True)
    del table
    orc = fn_oracle()
    otable = load(orc, s)
    per, rows, _ = run(orc, s, otable, args.oracle_steps, device=False)
    med = np.median(np.array(per), axis=0)
    print(json.dumps({"backend": "oracle", "live_keys": args.live, "commands": args.cmds, "steps": args.oracle_steps,
                      "commands_ms": round(med[0], 1), "delta_ms": round(med[1], 1), "insert_ms": round(med[2], 1),
                      "step_ms": round(float(sum(med)), 1), "delta_rows": rows, "card": name,
                      "power_limit_max_sm_clock": power}), flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--live", type=int, default=50_000_000)
    ap.add_argument("--cmds", type=int, default=5_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--oracle-steps", type=int, default=2)
    args = ap.parse_args()
    main()
