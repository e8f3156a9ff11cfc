"""The exchange model's placement (tests/exchange_model.py) against the oracle's shard_partition, row for row, on
full-range u64 / i64 lanes, 1 to 4 key lanes with value lanes, and worlds of 1 to 32 ranks.  This pins the model to
the oracle; tests/test_gpu_exchange.py then pins the CUDA exchange to the model."""
import numpy as np
import pytest

import edge_cases as ec
import exact_model as em
import exchange_model as xm
from dbsp_b200 import Schema

PLACEMENT_SCHEMAS = [Schema("u", "i"), Schema("i", "uu"), Schema("iu", "i"), Schema("uiu", "iu"), Schema("iiuu", "uuui"),
                     Schema("u"), Schema("ii")]
WORLDS = [1, 2, 3, 5, 8, 32]


def full_rows(schema, n, seed):
    rng = np.random.default_rng(seed)
    return ec.with_duplicates(rng, [ec.full_lane(rng, t, n, 0.4) for t in schema.lanes], ec.edge_weights(rng, n))


@pytest.mark.parametrize("schema", PLACEMENT_SCHEMAS, ids=ec.sid)
def test_placement_matches_oracle(oracle, schema):
    cols, w = full_rows(schema, 3000, 11 * schema.nk + schema.nv)
    b = oracle.batch_from_columns(schema, cols, w)
    for P in WORLDS:
        parts = oracle.shard_partition(b, P)
        want = xm.shard(schema, [(cols, w)], P)
        for p in range(P):
            em.assert_batch_is(parts[p], want[p], f"shard {p} of {P}, {ec.sid(schema)}")
        # rows that share a key share a rank, whatever their values
        if schema.nv:
            ccols, _ = xm.union(schema, [(cols, w)])
            d = xm.dests(ccols[: schema.nk], P)
            owner = {}
            for i in range(len(d)):
                k = tuple(int(c[i]) for c in ccols[: schema.nk])
                assert owner.setdefault(k, d[i]) == d[i]


@pytest.mark.parametrize("nk", [1, 2, 3, 4])
def test_int_and_numpy_placement_agree(nk):
    """dest_of (Python ints, the definition) == dests (numpy) on the extremes of both lane types and on random keys."""
    pool = sorted({em.u64(v) for v in ec.U_POOL + ec.I_POOL})
    rng = np.random.default_rng(nk)
    rows = [tuple(pool[(i * 3 + l * 5) % len(pool)] for l in range(nk)) for i in range(len(pool) ** 2)]
    rows += [tuple(int(x) for x in rng.integers(0, 1 << 64, nk, dtype=np.uint64)) for _ in range(500)]
    cols = [np.array([r[l] for r in rows], dtype=np.uint64) for l in range(nk)]
    for P in WORLDS:
        assert xm.dests(cols, P).tolist() == [xm.dest_of(r, P) for r in rows]


def test_mix64_known_values():
    """splitmix64's published output for seed 0 (the first three draws: mix64 of 1, 2, 3 golden-ratio steps)."""
    assert xm.mix64(0) == 0xE220A8397B1DCDAF
    assert xm.mix64(xm.GOLDEN) == 0x6E789E6AA1B965F4
    assert xm.mix64(2 * xm.GOLDEN & em.UMAX) == 0x06C45D188009454F


def test_round_model():
    """The model's own round arithmetic: union placement, gather, the unsigned maximum, the byte count."""
    s = Schema("i", "u")
    a = ([np.array([em.u64(em.MIN), 5], np.uint64), np.array([1, 2], np.uint64)], np.array([em.MIN, 3], np.int64))
    b = ([np.array([em.u64(em.MIN), 7], np.uint64), np.array([1, 2], np.uint64)], np.array([em.MIN, 4], np.int64))
    out = xm.shard(s, [a, b], 3)
    rows = sorted((int(c0), int(c1), int(w)) for cols, w in out for c0, c1, w in zip(cols[0], cols[1], w))
    assert rows == [(5, 2, 3), (7, 2, 4)]   # (MIN, 1) cancels: MIN + MIN = 0
    g = xm.gather(s, [a, b], 1, 2)
    assert len(g[0][1]) == 0 and len(g[1][1]) == 2
    assert xm.allreduce_max([0, (1 << 63) - 1, 1 << 63, -1]) == em.UMAX
    assert xm.allreduce_max([0, (1 << 63) - 1, 1 << 63]) == 1 << 63
    assert xm.bytes_sent(s, a, 0, 2, root=0) == 0 and xm.bytes_sent(s, a, 1, 2, root=0) == 2 * 3 * 8
    d = [xm.dest_of([em.u64(em.MIN)], 2), xm.dest_of([5], 2)]
    assert xm.bytes_sent(s, a, 0, 2) == sum(x != 0 for x in d) * 24
