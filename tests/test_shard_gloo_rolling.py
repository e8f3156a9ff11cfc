"""partitioned_rolling_aggregate on 2 and 3 workers (gloo, the CPU oracle with dbsp_rolling_aggregate): every worker
gets a slice of each step's rows, the stream is sharded by partition key, and the gathered integral of the output
must equal the non-incremental model at every step, in the plain and the watermark forms."""
import os
import socket
import sys

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def steps():
    r = np.random.default_rng(31)
    return [[(int(p), int(t), int(v), int(w)) for p, t, v, w in
             zip(r.integers(0, 7, 60), r.integers(i * 50, i * 50 + 400, 60), r.integers(-50, 50, 60), r.choice([-1, 1, 1, 2], 60))]
            for i in range(8)]


def _worker(rank, world, port, outdir):
    for p in (ROOT, HERE):
        if p not in sys.path:
            sys.path.insert(0, p)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import rolling_cases as rc
    from dbsp_b200.parallel import Comm
    from rowfn_cases import fn_oracle

    results = []
    for lateness in (None, 300):
        c, h, outs = rc.build(fn_oracle(), rc.REF_SCHEMA, rc.REF_AGGS, rc.REF_RANGES[1], lateness, Comm())
        for rows in steps():
            h.append([rows[i] for i in np.array_split(np.arange(len(rows)), world)[rank]])
            c.step()
            if rank == 0:
                results.append([integ.value.rows() for _, _, integ, _ in outs])
    if rank == 0:
        np.save(os.path.join(outdir, "sharded.npy"), np.array(results, dtype=object), allow_pickle=True)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_rolling_equal_model(tmp_path, world):
    import rolling_cases as rc
    from rowfn_cases import fn_oracle

    fn_oracle()   # built here, before the workers load it
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    sharded = np.load(os.path.join(tmp_path, "sharded.npy"), allow_pickle=True)
    k = 0
    for _ in (None, 300):
        integral = {}
        for i, rows in enumerate(steps()):
            rc._integrate(integral, rows)
            for a, got in zip(rc.REF_AGGS, sharded[k]):
                want = rc.model(integral, rc.REF_SCHEMA, rc.REF_RANGES[1], a.kind, a.py, a.f_types)
                assert rc._as_dict(got) == want, f"step {i} {a.kind}"
            k += 1
