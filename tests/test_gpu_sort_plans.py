"""Consolidation past 5 M rows, on every sort plan of csrc/sort.cu: splitters at 8 K, 16 K and 32 K buckets on both
sides of each bucket-count boundary, plain LSD above MAX_BUCKETS * 768 rows, chunk-only sorts of rows whose lane 0
arrives ordered, the LSD fallback after a bucket overflows a chunk, wide rows sorted word by word, the sort-free
paths of ordered rows, and the epilogue's look-backs across more than 65 536 tiles.  Every case is compared bit for
bit with the numpy model (exact_model.consolidate_np) and asserts the plan that ran (sort_plan_cases.check_plan).

Each case runs on a context of its own that is destroyed when the case ends, so the few GiB a case needs go back
to the device instead of staying in the pool of the session's context."""
import numpy as np
import pytest

import sort_plan_cases as sp
from dbsp_b200 import Schema
from exact_model import assert_batch_is, consolidate_np

pytestmark = pytest.mark.gpu


@pytest.fixture
def be():
    import dbsp_b200.runtime as rt

    r = rt.Runtime(0)
    yield r
    r.sync()
    r.close()


def check(be, what, call, schema, cols, w, want):
    """call() consolidates the rows (cols, w) of `schema`, in that order: the plan it ran is `want`, its batch is
    the model's"""
    n = len(w)
    kp = sp.KeyPlan(schema, cols, w)
    be.profile(True)
    b = call()
    prof = be.profile_read()
    be.profile(False)
    assert_batch_is(b, consolidate_np(schema, cols, w), what)
    sp.check_plan(prof, n, kp, want, what)
    del b
    be.sync()


def from_columns(be, what, schema, cols, w, want):
    check(be, what, lambda: be.batch_from_columns(schema, cols, w), schema, cols, w, want)


def want_for(n):
    return "lsd" if n > sp.LSD_MAX_ROWS else f"splitters({sp.n_buckets(n)})"


@pytest.mark.parametrize("n", [6_291_456, 6_291_457, 12_582_912, 12_582_913, 25_165_824, 25_165_825, 40_000_003])
def test_one_word_bucket_boundaries(be, n):
    """nb * 768 and nb * 768 + 1 rows for nb = 8 K, 16 K, 32 K; 32 K * 768 + 1 and 40 M rows take plain LSD"""
    from_columns(be, f"one word, n={n}", *sp.one_word(n, n), want_for(n))


@pytest.mark.parametrize("n", [20_000_000, 30_000_000])
@pytest.mark.parametrize("dist", sp.DISTS)
def test_key_distributions(be, n, dist):
    from_columns(be, f"{dist}, n={n}", *sp.distribution(n, dist, n % 997 + len(dist)), want_for(n))


@pytest.mark.parametrize("dups", [False, True])
def test_ordered_rows_are_not_sorted(be, dups):
    """30 M ordered rows: distinct with non-zero weights, the uploaded buffer becomes the batch (no pack, no sort, no
    epilogue); with duplicates and zero weights, one identity-order epilogue"""
    from_columns(be, f"ordered, dups={dups}", *sp.ordered_rows(30_000_000, dups, 5), "ordered" if dups else "adopted")


@pytest.mark.parametrize("n,run,want", [(20_000_000, 0, "splitters(32768)"), (30_000_000, 0, "lsd"),
                                        (30_000_000, 920, "chunks"), (30_000_000, 9200, "chunks -> lsd fallback")])
def test_two_word_keys(be, n, run, want):
    """q7's row shape (two key words, an aliased lane).  run > 0: lane 0 arrives ordered in runs of `run` rows;
    920-row runs are chunk-only over ~32 K windows, 9 200-row runs (q7 at 10 M events/s) overflow a chunk"""
    schema, cols, w = sp.q7_rows(n, n + run, run)
    kp = sp.KeyPlan(schema, cols, w)
    assert kp.W == 2 and kp.bits[3] == 0, (kp.W, kp.bits)
    from_columns(be, f"q7 rows, n={n}, run={run}", schema, cols, w, want)


@pytest.mark.parametrize("two_words", [False, True])
def test_sample_defeating_rows_fall_back(be, two_words):
    """The smallest row at every sampled row: all splitters are equal, one bucket holds almost every row"""
    n = 20_000_000
    schema, cols, w = sp.sample_defeating(n, 11, two_words)
    assert sp.KeyPlan(schema, cols, w).W == (2 if two_words else 1)
    from_columns(be, f"sample-defeating rows, two_words={two_words}", schema, cols, w, "splitters(32768) -> lsd fallback")


@pytest.mark.parametrize("n,defeat,want", [(8_000_000, False, "splitters(16384)"), (30_000_000, False, "lsd"),
                                           (8_000_000, True, "splitters(16384) -> lsd fallback")])
def test_wide_rows_sorted_word_by_word(be, n, defeat, want):
    """Three key words, one sort per word: stability decides the order of rows equal in lanes 0 and 1.  defeat:
    word 0's sort overflows a chunk and leaves its row ids half-written, word 1 is packed through them, then every
    word is sorted again by LSD"""
    schema, cols, w = sp.wide_rows(n, n + defeat, defeat)
    assert sp.KeyPlan(schema, cols, w).W == 3
    from_columns(be, f"wide rows, n={n}, defeat_word0={defeat}", schema, cols, w, "3 words, " + want)


def test_epilogue_lookback_over_68k_tiles(be):
    """70 M rows (68 360 epilogue tiles of 1 024 rows): a run of 5 M equal rows whose weights sum to 0 and one whose
    weights sum to i64::MIN, each spanning ~4 900 tiles"""
    schema, cols, w = sp.cancelling_runs(70_000_000, 5_000_000, 3)
    from_columns(be, "70 M rows", schema, cols, w, "lsd")


@pytest.mark.parametrize("n", [400_000, 1_000_000])
def test_fanout_table_over_lsd_threshold(be, n):
    """batch_from_table with a 64-way fan-out: 25.6 M and 64 M rows"""
    cols, w, proj, schema, mcols, mw = sp.fanout_table(n, n)
    check(be, f"fan-out table n={n}", lambda: be.batch_from_table(cols, proj, w), schema, mcols, mw, "lsd")


def test_fanout_map_index_over_lsd_threshold(be):
    """map_index with a 32-way fan-out over a 1 M-row batch: 32 M rows"""
    rng = np.random.default_rng(8)
    s, n = Schema("u", "u"), 1_000_000
    cols = [rng.integers(0, 1 << 20, n).astype(np.uint64), rng.integers(0, 1 << 18, n).astype(np.uint64)]
    w = rng.choice(np.array([-2, -1, 1, 2]), n)
    inp, rows = be.batch_from_columns(s, cols, w), consolidate_np(s, cols, w)
    assert_batch_is(inp, rows, "map_index input")
    proj, mcols, mw = sp.fanout_map(rows)
    check(be, "fan-out map_index", lambda: be.map_index(inp, proj), proj.schema, mcols, mw, "lsd")


def test_join_output_over_lsd_threshold(be):
    """join_batches with 5 000 keys x 100 left x 60 right rows: 30 M output rows"""
    lc, lw, rc, rw, proj, (mcols, mw) = sp.join_sides(5000, 100, 60, 4)
    s = Schema("u", "u")
    left, right = be.batch_from_columns(s, lc, lw), be.batch_from_columns(s, rc, rw)
    check(be, "join output", lambda: be.join_batches(left, right, proj), proj.schema, mcols, mw, "lsd")
