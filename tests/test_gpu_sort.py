"""The hand-written radix sort inside Batch::from_tuples (csrc/sort.cu) against the oracle's comparison sort, across
its plans: single shared-memory chunk, top-digit HBM passes + chunks, presorted leading lane (no HBM pass), the plain
LSD fallback after the skew flag, multi-word keys."""
import numpy as np
import pytest

import sort_plan_cases as sp
from dbsp_b200 import Schema
from parity_util import assert_batches_equal

pytestmark = pytest.mark.gpu


def check(cuda, oracle, schema, cols, w, what):
    assert_batches_equal(cuda.batch_from_columns(schema, cols, w), oracle.batch_from_columns(schema, cols, w), what)


@pytest.mark.parametrize("n", [2, 31, 33, 3071, 3072, 3073, 6143, 6144, 6145, 9217, 60_000, 1_000_003, 4_600_000])
@pytest.mark.parametrize("bits", [3, 17, 40, 63])
def test_sort_sizes_and_widths(cuda, oracle, n, bits):
    rng = np.random.default_rng(n * 7 + bits)
    s = Schema("u", "u")
    hi = max(bits - 20, 1)
    cols = [rng.integers(0, 1 << hi, n).astype(np.uint64), rng.integers(0, 1 << (bits - hi + 1), n).astype(np.uint64)]
    check(cuda, oracle, s, cols, rng.integers(-2, 3, n), f"n={n} bits={bits}")


@pytest.mark.parametrize("n", [50_000, 2_000_000])
def test_sort_skew_falls_back(cuda, oracle, n):
    """One hot key holds 70 % of the rows.  Below 256 K rows its top-digit bucket cannot fit a chunk and the LSD
    fallback takes over; at 2 M rows the hot rows still differ in their 33-bit value lane, so the splitters divide
    them and no bucket overflows.  A single key with random values sorts without a fallback, and rows that are all
    equal arrive ordered and are not sorted at all.  The profile shows which plan each ran."""
    hot_plan, single_plan = {50_000: ("top digit -> lsd fallback", "top digit"), 2_000_000: ("splitters(4096)",) * 2}[n]
    rng = np.random.default_rng(n)
    s = Schema("u", "u")
    k = np.where(rng.random(n) < 0.7, 12345, rng.integers(0, 1 << 30, n)).astype(np.uint64)
    v = rng.integers(0, 1 << 33, n).astype(np.uint64)
    for what, cols, w, plan in [("hot key", [k, v], rng.integers(-1, 2, n), hot_plan),
                                ("single key", [np.full(n, 7, np.uint64), v], np.ones(n, np.int64), single_plan),
                                ("single row", [np.full(n, 7, np.uint64), np.full(n, 9, np.uint64)], np.ones(n, np.int64), "ordered")]:
        cuda.profile(True)
        check(cuda, oracle, s, cols, w, what)
        prof = cuda.profile_read()
        cuda.profile(False)
        sp.check_plan(prof, n, sp.KeyPlan(s, cols, w), plan, what)


@pytest.mark.parametrize("run", [1, 9, 900, 3000, 3073, 20_000])
def test_sort_presorted_leading_lane(cuda, oracle, run):
    """Lane 0 arrives ordered (time-ordered event tables) with equal-lane-0 runs of `run` rows: short runs take the
    no-HBM-pass path, runs longer than half a chunk raise the flag."""
    n = 700_000
    rng = np.random.default_rng(run)
    s = Schema("u", "uuu")
    t = (np.arange(n) // run).astype(np.uint64) + np.uint64(1_000_000)
    cols = [t, rng.integers(0, 5000, n).astype(np.uint64), rng.integers(0, 1 << 20, n).astype(np.uint64), rng.integers(0, 3, n).astype(np.uint64)]
    check(cuda, oracle, s, cols, rng.integers(-1, 2, n), f"run={run}")


def test_sort_multiword(cuda, oracle):
    rng = np.random.default_rng(3)
    n = 800_000
    s = Schema("ui", "uuu")
    cols = [rng.integers(0, 1 << 50, n).astype(np.uint64), rng.integers(-(1 << 40), 1 << 40, n), rng.integers(0, 1 << 30, n).astype(np.uint64),
            rng.integers(0, 1 << 62, n).astype(np.uint64), rng.integers(0, 4, n).astype(np.uint64)]
    for c in cols[:2]:
        c[n // 2:] = c[: n - n // 2]   # equal leading lanes: the low words decide
    check(cuda, oracle, s, cols, rng.integers(-1, 2, n), "three words")


@pytest.mark.parametrize("n", [262_143, 262_144, 700_001, 3_000_000])
@pytest.mark.parametrize("dist", ["uniform", "loguniform", "hitters", "fewvalues"])
def test_sort_splitter_mode(cuda, oracle, n, dist):
    """n >= 256 K rows: bucket ids from sampled splitters, whatever the key distribution (log-uniform prices put a
    quarter of the rows under one top-bits prefix; heavy hitters end up in equality buckets that need no sorting)."""
    rng = np.random.default_rng(n % 1000 + len(dist))
    s = Schema("u", "uu")
    if dist == "uniform":
        k = rng.integers(0, 1 << 40, n)
    elif dist == "loguniform":
        k = np.ceil(np.power(10.0, rng.random(n) * 6.0) * 100.0).astype(np.int64)
    elif dist == "hitters":
        k = np.where(rng.random(n) < 0.6, rng.choice(np.array([5, 77, 1 << 33]), n), rng.integers(0, 1 << 35, n))
    else:
        k = rng.integers(0, 7, n)
    cols = [k.astype(np.uint64), rng.integers(0, 1 << 18, n).astype(np.uint64), rng.integers(0, 50, n).astype(np.uint64)]
    check(cuda, oracle, s, cols, rng.integers(-1, 3, n), f"splitters n={n} {dist}")


@pytest.mark.parametrize("n", [5_000, 200_000, 2_000_000])
def test_sort_two_word_keys(cuda, oracle, n):
    """Rows wider than 64 packed bits (two key words): one sort over the whole key, the epilogue unpacks both words."""
    rng = np.random.default_rng(n)
    s = Schema("u", "uuuuu")   # the shape of q7's bids_by_price: (price, auction, bidder, price, date_time, extra)
    price = np.ceil(np.power(10.0, rng.random(n) * 6.0) * 100.0).astype(np.uint64)
    cols = [price, rng.integers(1000, 300_000, n).astype(np.uint64), rng.integers(1000, 100_000, n).astype(np.uint64), price,
            (np.uint64(1436918400000) + rng.integers(0, 10_000, n).astype(np.uint64)), rng.integers(0, 1 << 32, n).astype(np.uint64)]
    # exact duplicates and cancelling pairs
    for c in cols:
        c[: n // 10] = c[n // 10: 2 * (n // 10)]
    w = rng.integers(-1, 2, n)
    check(cuda, oracle, s, cols, w, f"two words n={n}")


def test_sort_two_word_presorted(cuda, oracle):
    """Time-ordered table with rows wider than one word (q7's bids_by_time): no HBM pass, two-word chunk sort."""
    n = 1_500_000
    rng = np.random.default_rng(9)
    s = Schema("u", "uuuu")
    t = np.uint64(1436918400000) + (np.arange(n) // 920).astype(np.uint64)
    price = np.ceil(np.power(10.0, rng.random(n) * 6.0) * 100.0).astype(np.uint64)
    cols = [t, rng.integers(1000, 300_000, n).astype(np.uint64), rng.integers(1000, 100_000, n).astype(np.uint64), price,
            rng.integers(0, 1 << 32, n).astype(np.uint64)]
    check(cuda, oracle, s, cols, np.ones(n, np.int64), "two words, presorted lane 0")


def test_sort_aliased_lanes(cuda, oracle):
    """A lane that repeats an earlier lane in every row is left out of the key and restored on unpack (q7's
    (price, auction, bidder, price, date_time, extra)); one differing row must disable the shortcut."""
    rng = np.random.default_rng(12)
    n = 400_000
    s = Schema("u", "uuuuu")
    price = np.ceil(np.power(10.0, rng.random(n) * 6.0) * 100.0).astype(np.uint64)
    base = [price, rng.integers(1000, 300_000, n).astype(np.uint64), rng.integers(1000, 100_000, n).astype(np.uint64), price.copy(),
            np.uint64(1436918400000) + rng.integers(0, 10_000, n).astype(np.uint64), rng.integers(0, 1 << 32, n).astype(np.uint64)]
    w = rng.integers(-1, 2, n)
    check(cuda, oracle, s, base, w, "lane 3 == lane 0")
    almost = [c.copy() for c in base]
    almost[3][n // 2] += np.uint64(1)
    check(cuda, oracle, s, almost, w, "lane 3 differs from lane 0 in one row")
    three = [c.copy() for c in base]
    three[2] = three[1].copy()   # lane 2 == lane 1 as well
    check(cuda, oracle, Schema("uu", "iuuu"), three, w, "two aliased lanes, mixed types")
