"""add_input_map / add_input_set on 2 and 3 workers (gloo, the CPU oracle with the upsert calls): each worker's
command batch is sharded by key before it meets the table's trace.  Whether every command goes to rank 0 or the
step's command list is cut into contiguous slices in rank order, the gathered output must equal the single-worker
output at every step: a key's commands are ordered by worker rank, then push order."""
import os
import socket
import sys

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
STEPS = 8


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def commands():
    """Per step: map commands (key, value or None) and set commands (key, bool) over a small key range, so that a
    key often has several commands in one step."""
    rng = np.random.default_rng(21)
    out = []
    for _ in range(STEPS):
        n = 3000
        mk = rng.integers(-300, 300, n)
        mv = rng.integers(0, 5, n)
        md = rng.random(n) < 0.25
        sk = rng.integers(0, 200, (n, 2))
        si = rng.random(n) < 0.6
        out.append(([(int(k), None if d else (int(v), -int(v))) for k, v, d in zip(mk, mv, md)],
                    [((int(a), int(b)), bool(i)) for (a, b), i in zip(sk, si)]))
    return out


def build(be, comm=None):
    from dbsp_b200 import RootCircuit, Schema

    c = RootCircuit(be, comm)
    m, hm = c.add_input_map(Schema("i", "ui"))
    s, hs = c.add_input_set(Schema("uu"))
    outs = [m, s]
    if comm is not None:
        outs = [o.gather(0) for o in outs]
    return c, (hm, hs), [o.output() for o in outs]


def my_slice(cmds, rank, world, split):
    if not split:
        return cmds if rank == 0 else []
    return [cmds[i] for i in np.array_split(np.arange(len(cmds)), world)[rank]]


def _worker(rank, world, port, outdir, split):
    for p in (ROOT, HERE):
        if p not in sys.path:
            sys.path.insert(0, p)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from dbsp_b200.parallel import Comm
    from rowfn_cases import fn_oracle

    c, (hm, hs), outs = build(fn_oracle(), Comm())
    results = []
    for mc, sc in commands():
        hm.append(my_slice(mc, rank, world, split))
        hs.append(my_slice(sc, rank, world, split))
        c.step()
        if rank == 0:
            results.append([o.value.rows() for o in outs])
    if rank == 0:
        np.save(os.path.join(outdir, "sharded.npy"), np.array(results, dtype=object), allow_pickle=True)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("split", [False, True], ids=["rank0", "slices"])
def test_sharded_upsert_equal_single(tmp_path, world, split):
    from rowfn_cases import fn_oracle

    be = fn_oracle()   # built here, before the workers load it
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path), split), nprocs=world, join=True)
    sharded = np.load(os.path.join(tmp_path, "sharded.npy"), allow_pickle=True)
    c, (hm, hs), outs = build(be)
    for i, (mc, sc) in enumerate(commands()):
        hm.append(mc)
        hs.append(sc)
        c.step()
        got = [o.value.rows() for o in outs]
        assert all(got), f"step {i}: an output is empty"
        for name, a, b in zip(("map", "set"), got, sharded[i]):
            assert a == list(b), f"{name} step {i}"
