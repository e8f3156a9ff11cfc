"""An exact model of one exchange round between P circuit replicas (include/dbsp_b200.h "communication"):
`dbsp_shard`, `dbsp_shard2`, `dbsp_gather`, `dbsp_allreduce_max_u64` and the byte count of `dbsp_comm_info`.

Placement restates DESIGN §2 "Shard hash": the splitmix64 fold over the KEY lanes only, h = 0, h = mix64(h ^ lane),
destination h % P.  It shares no code with the library or the oracle.  `dest_of` is the definition in Python ints;
`dests` is the same fold on numpy uint64 columns for large batches (tests/test_exchange_model.py pins the two
together and both to the oracle's placement).  Consolidation is exact_model's.

A rank's input is (cols, weights): numpy uint64 columns and int64 weights, as given to `batch_from_columns`; the
model consolidates it first, as the replica does when it builds its batch."""
import numpy as np

import exact_model as em
from exact_model import UMAX

GOLDEN = 0x9E3779B97F4A7C15


def mix64(x):
    """splitmix64's finaliser on a Python int in [0, 2^64)."""
    x = (x + GOLDEN) & UMAX
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & UMAX
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & UMAX
    return x ^ (x >> 31)


def dest_of(key_lanes, P):
    """The rank that owns a key: key_lanes are the key's lanes (typed ints or u64 bit patterns)."""
    h = 0
    for k in key_lanes:
        h = mix64(h ^ em.u64(int(k)))
    return h % P


def _mix64_np(x):
    with np.errstate(over="ignore"):
        x = x + np.uint64(GOLDEN)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def dests(key_cols, P):
    """dest_of for every row of numpy key columns (uint64 bit patterns): an int64 array."""
    n = len(key_cols[0])
    h = np.zeros(n, np.uint64)
    for c in key_cols:
        h = _mix64_np(h ^ np.asarray(c).view(np.uint64))
    return (h % np.uint64(P)).astype(np.int64)


def _empty(schema):
    return [np.zeros(0, np.uint64) for _ in range(schema.nl)], np.zeros(0, np.int64)


def consolidated(schema, inp):
    cols, w = inp
    return em.consolidate_np(schema, [np.asarray(c).view(np.uint64) for c in cols], w)


def _concat(schema, parts):
    cols = [np.concatenate([p[0][l] for p in parts]) for l in range(schema.nl)]
    return cols, np.concatenate([p[1] for p in parts])


def union(schema, inputs):
    """The consolidated union of the ranks' (consolidated) inputs."""
    return em.consolidate_np(schema, *_concat(schema, [consolidated(schema, i) for i in inputs]))


def shard(schema, inputs, P):
    """dbsp_shard: the output of every rank, [(cols, weights)] * P, each the consolidated union of the rows whose
    key hashes to that rank."""
    cols, w = union(schema, inputs)
    d = dests(cols[: schema.nk], P) if len(w) else np.zeros(0, np.int64)
    return [([c[d == r] for c in cols], w[d == r]) for r in range(P)]


def gather(schema, inputs, root, P):
    """dbsp_gather: the union on `root`, empty batches elsewhere."""
    return [union(schema, inputs) if r == root else _empty(schema) for r in range(P)]


def allreduce_max(values):
    """dbsp_allreduce_max_u64: the unsigned maximum, handed to every rank."""
    return max(em.u64(int(v)) for v in values)


def bytes_sent(schema, inp, rank, P, root=None):
    """Payload bytes one round adds to `rank`'s dbsp_comm_info count: (L+1)*8 for every row of its consolidated
    input that goes to another rank (all rows to `root` for a gather)."""
    cols, w = consolidated(schema, inp)
    if root is not None:
        away = 0 if root == rank else len(w)
    else:
        away = int(np.count_nonzero(dests(cols[: schema.nk], P) != rank)) if len(w) else 0
    return away * (schema.nl + 1) * 8


def keys_with_dest(rng, n_key_lanes, P, per_dest):
    """Random 64-bit keys sorted by owner: for every rank p, `per_dest` (or per_dest[p]) key tuples (one uint64
    column per key lane) that hash to p.  (Two of them are equal with negligible probability; the model would sum
    them anyway.)"""
    want = list(per_dest) if isinstance(per_dest, (list, tuple)) else [per_dest] * P
    got = [[[] for _ in range(n_key_lanes)] for _ in range(P)]
    while any(w > 0 for w in want):
        n = 2 * P * max(want) + 64
        cols = [rng.integers(0, 1 << 64, n, dtype=np.uint64) for _ in range(n_key_lanes)]
        d = dests(cols, P)
        for p in range(P):
            idx = np.flatnonzero(d == p)[: max(want[p], 0)]
            for l, c in enumerate(cols):
                got[p][l].append(c[idx])
            want[p] -= len(idx)
    return [[np.concatenate(g) for g in got[p]] for p in range(P)]
