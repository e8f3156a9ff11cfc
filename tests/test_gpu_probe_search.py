"""The per-batch key search of the join probe and of the Max / Min walk: a warp's 32 consecutive keys skip the
batches their span misses, narrow a shared window in the others, then search their own range inside it.  Every case
compares `join_delta_trace` (delta on either side) and Max / Min `aggregate_delta` with the exact model
(tests/exact_model.py) and bit for bit with the CPU oracle, at the places where that search can go wrong: keys at a
batch's first and last key and one beside them, spans below, above and between the batches, batches whose ranges
interleave, partial warps, multi-lane and signed keys at MIN / MAX, one key of more than 1024 matches, totals just
past a fill tile, truncated spines, and more than 16 batches (one launch takes 16)."""
import itertools

import numpy as np
import pytest

import exact_model as em
from dbsp_b200 import Proj, Schema, Spine, capi, key, lval, rval
from exact_model import MAX, MIN, UMAX, Z
from parity_util import assert_batches_equal

pytestmark = pytest.mark.gpu

# sorted distinct key tuples of each key schema (~3000), extremes included
UNIVERSE = {
    "i": sorted({MIN, MIN + 1, MAX - 1, MAX} | set(range(-1500, 1500))),
    "uu": sorted(itertools.product([0, 1, 5, 1 << 63, UMAX - 1, UMAX], range(500))),
    "iui": sorted(itertools.product([MIN, -1, 0, MAX], [0, UMAX], [MIN] + list(range(-200, 200)) + [MAX])),
}
UNIVERSE["i"] = [(k,) for k in UNIVERSE["i"]]


def key_rows(ks, spans, seed, vt="u"):
    """One batch per (first, last, n) span of universe indices: n rows cycling over the span's keys, every row's value
    distinct, weights in {-2, -1, 1, 2, 3}."""
    U = UNIVERSE[ks]
    rng = np.random.default_rng(seed)
    out = []
    for b, (first, last, n) in enumerate(spans):
        span = last - first + 1
        vals = [(b << 40) + j for j in range(n)]
        if vt == "i":   # signed values reach MIN and MAX
            vals = [MIN + v if j % 2 else MAX - v for j, v in enumerate(vals)]
        w = rng.choice([-2, -1, 1, 2, 3], n)
        out.append([U[first + j % span] + (vals[j], int(w[j])) for j in range(n)])
    return out


def spines(bes, schema, batches, trunc=None):
    """One spine per backend holding `batches` (rows) in order, truncated below universe key `trunc` if given, and
    the model of their union."""
    sps, z = [Spine(b, schema) for b in bes], Z(schema)
    for rows in batches:
        for sp, b in zip(sps, bes):
            sp.insert(b.batch_from_rows(schema, rows))
        z.add(rows)
    if trunc is not None:
        for sp in sps:
            sp.truncate_keys_below(trunc)
        z = em.truncate_keys_below(z, trunc)
    return sps, z


def delta_rows(ks, idx, seed):
    """1-3 rows on each universe index of `idx` (out-of-range indices dropped)."""
    U = UNIVERSE[ks]
    rng = np.random.default_rng(seed)
    rows = []
    for i in sorted({i for i in idx if 0 <= i < len(U)}):
        for r in range(int(rng.integers(1, 4))):
            rows.append(U[i] + (int(rng.integers(0, 1 << 64, dtype=np.uint64)), int(rng.choice([-1, 1, 2]))))
    return rows


def check_join(cuda, oracle, ks, sps, zt, rows, what):
    nk = len(ks)
    ds = Schema(ks, "u")
    proj = Proj(Schema(ks, "uu"), [key(l) for l in range(nk)] + [lval(0), rval(0)])
    for left in (True, False):
        exp = em.join_delta_trace(Z(ds, rows), zt, proj, delta_is_left=left)
        got = cuda.join_delta_trace(cuda.batch_from_rows(ds, rows), sps[0], proj, delta_is_left=left)
        other = oracle.join_delta_trace(oracle.batch_from_rows(ds, rows), sps[1], proj, delta_is_left=left)
        w = f"join {what} left={left}"
        em.assert_batch_is(got, exp, w)
        assert_batches_equal(got, other, f"{w}: vs oracle")


def check_extremum(cuda, oracle, ks, spans, rows, what, trunc=None):
    """Max and Min of the keys of `rows`, inserted as the newest batch of an in-trace of `spans` (signed values)."""
    s = Schema(ks, "i")
    base = key_rows(ks, spans, 5, vt="i")
    rows = [r[:-2] + (em.w64(r[-2]), r[-1]) for r in rows]
    if trunc is not None:   # a truncated spine drops later inserts below the cut too
        rows = [r for r in rows if r[: len(ks)] >= tuple(trunc)]
    for kind in (capi.AGG_MAX, capi.AGG_MIN):
        sps, zin = spines([cuda, oracle], s, base, trunc)
        outs = [Spine(b, s) for b in (cuda, oracle)]
        delta = Z(s, rows)
        zin.add(delta.rows())
        exp = em.aggregate_delta(delta, zin, Z(s), kind)
        res = []
        for sp, osp, b in zip(sps, outs, (cuda, oracle)):
            d = b.batch_from_rows(s, rows)
            sp.insert(d)
            res.append(b.aggregate_delta(d, sp, osp, kind))
        w = f"aggregate kind {kind} {what} over {sps[0].stats()[1]} batches"
        em.assert_batch_is(res[0], exp, w)
        assert_batches_equal(res[0], res[1], f"{w}: vs oracle")


# Batches of shrinking size (so the spine keeps them apart): two that interleave, one above them, one at each end of
# the universe, and one narrow batch far above; the gaps between them hold no key.
def layout(N):
    return [(100, 1099, 6000), (600, 1699, 2500), (1500, 1799, 900), (0, 40, 300), (N - 41, N - 1, 120),
            (2500, 2509, 40)]


def edge_keys(spans, N):
    idx = [0, 1, 2, N - 1, N - 2, 1800, 1900, 2000, 2200, 2400, 2510, 2600]   # ends, between and above the batches
    for first, last, _ in spans:
        idx += [first - 1, first, first + 1, last - 1, last, last + 1]
    return idx


def key_sets(N, spans):
    rng = np.random.default_rng(3)
    sets = {"edges": edge_keys(spans, N)}
    for n in (1, 31, 32, 33):   # partial and full warps, a key alone
        sets[f"{n}_at_batch_start"] = list(range(600 - n // 2, 600 - n // 2 + n))
        sets[f"{n}_above_all"] = list(range(2700, 2700 + n))
    sets["1_last"] = [N - 1]
    sets["1200_random"] = rng.choice(N, 1200, replace=False).tolist()
    return sets


@pytest.mark.parametrize("ks", list(UNIVERSE))
def test_probe_search_edges(cuda, oracle, ks):
    N = len(UNIVERSE[ks])
    spans = layout(N)
    sps, zt = spines([cuda, oracle], Schema(ks, "u"), key_rows(ks, spans, 1))
    assert sps[0].stats()[1] >= 4, sps[0].stats()
    for name, idx in key_sets(N, spans).items():
        rows = delta_rows(ks, idx, 7)
        check_join(cuda, oracle, ks, sps, zt, rows, f"{ks} {name}")
        check_extremum(cuda, oracle, ks, spans, rows, f"{ks} {name}")


@pytest.mark.parametrize("total", [255, 256, 257, 1025, 2047, 3000])
def test_probe_fill_tiles(cuda, oracle, total):
    """One key of `total` matches split over two batches (more than 1024 from 1025 on): alone, so the fill's total is
    just past or at a tile boundary, and after 200 keys of 300 matches, so its run starts inside a tile."""
    ks = "i"
    hot = total - total // 3
    spans = [(0, 199, 300), (1000, 1000, hot), (1000, 1000, total - hot)]
    sps, zt = spines([cuda, oracle], Schema(ks, "u"), key_rows(ks, spans, 11))
    U = UNIVERSE[ks]
    for name, rows in {"alone": [U[1000] + (7, 1)], "after": [U[i] + (i, 1) for i in list(range(200)) + [1000]]}.items():
        check_join(cuda, oracle, ks, sps, zt, rows, f"hot key of {total} matches {name}")
        check_extremum(cuda, oracle, ks, spans, rows, f"hot key of {total} values {name}")


@pytest.mark.parametrize("ks", ["i", "iui"])
def test_probe_search_truncated(cuda, oracle, ks):
    """A spine truncated below a key inside the interleaving batches: the searches start at the kept rows."""
    N = len(UNIVERSE[ks])
    spans = layout(N)
    trunc = UNIVERSE[ks][650]
    sps, zt = spines([cuda, oracle], Schema(ks, "u"), key_rows(ks, spans, 2), trunc)
    for name, idx in {"edges": edge_keys(spans, N) + [649, 650, 651], "around_cut": list(range(630, 700))}.items():
        rows = delta_rows(ks, idx, 9)
        check_join(cuda, oracle, ks, sps, zt, rows, f"truncated {ks} {name}")
        check_extremum(cuda, oracle, ks, spans, rows, f"truncated {ks} {name}", trunc)


def test_probe_search_deep(cuda, oracle):
    """18 batches of halving size over overlapping key spans: the join probes them in two launches."""
    ks = "uu"
    N = len(UNIVERSE[ks])
    spans = [(i * 150, i * 150 + 199, 1 << (17 - i)) for i in range(18)]
    sps, zt = spines([cuda, oracle], Schema(ks, "u"), key_rows(ks, spans, 4))
    assert sps[0].stats()[1] > 16, sps[0].stats()
    idx = [i for first, last, _ in spans for i in (first - 1, first, last, last + 1)] + [N - 1, N - 3]
    rows = delta_rows(ks, idx, 13)
    check_join(cuda, oracle, ks, sps, zt, rows, "18 batches")
    check_extremum(cuda, oracle, ks, spans[8:], rows, "10 batches")
