"""aggregate(Fold) and Nexmark q18 on two workers (world_size-2 gloo, the CPU oracle with dbsp_aggregate_fold): the
sharded circuit's gathered output must equal the single-worker output, step by step.  Each worker folds the keys it
owns after the shard; rows arrive round-robin, so every key's values are split across the workers before the
exchange, and a key's walk must see all of them in value order."""
import os
import socket
import sys

import numpy as np
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
N_EVENTS, STEP = 120_000, 30_000


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def build(be, comm=None):
    """Per step: q18, and a weighted fold of the bids' prices per auction (aggregate(Fold) reading the weight)."""
    from dbsp_b200 import Proj, RootCircuit, Schema, col
    from dbsp_b200.nexmark import queries as nq
    import fold_cases as fc

    c = RootCircuit(be, comm)
    inp, handles = nq.add_nexmark_input(c)
    prices = inp.bid.flat_map_index(Proj(Schema("u", "ii"), [col(0), col(2), col(1)]))
    outs = [nq.q18(inp), prices.aggregate(fc.f_weight())]
    if comm is not None:
        outs = [o.gather(0) for o in outs]
    return c, handles, [o.output() for o in outs]


def tables(gen, s0, rank=0, world=1):
    t = gen.tables(s0, STEP)
    return {k: [col[rank::world].copy() for col in v] for k, v in t.items()}   # round-robin input (input.rs:664-703)


def _worker(rank, world, port, outdir):
    for p in (ROOT, HERE):
        if p not in sys.path:
            sys.path.insert(0, p)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from dbsp_b200.nexmark import NexmarkGenerator
    from dbsp_b200.parallel import Comm
    from rowfn_cases import fn_oracle

    c, handles, outs = build(fn_oracle(), Comm())
    gen = NexmarkGenerator(first_event_rate=1)
    results = []
    for s0 in range(0, N_EVENTS, STEP):
        for k, v in tables(gen, s0, rank, world).items():
            handles[k].set(v)
        c.step()
        if rank == 0:
            results.append([o.value.rows() for o in outs])
    if rank == 0:
        np.save(os.path.join(outdir, "sharded.npy"), np.array(results, dtype=object), allow_pickle=True)
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_fold_equal_single(tmp_path):
    from dbsp_b200.nexmark import NexmarkGenerator
    from rowfn_cases import fn_oracle

    be = fn_oracle()   # built here, before the workers load it
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    sharded = np.load(os.path.join(tmp_path, "sharded.npy"), allow_pickle=True)
    c, handles, outs = build(be)
    gen = NexmarkGenerator(first_event_rate=1)
    for i, s0 in enumerate(range(0, N_EVENTS, STEP)):
        for k, v in tables(gen, s0).items():
            handles[k].set(v)
        c.step()
        got = [o.value.rows() for o in outs]
        assert all(got), f"step {i}: an output is empty"
        for name, a, b in zip(("q18", "aggregate(Fold)"), got, sharded[i]):
            assert a == list(b), f"{name} step {i}"
