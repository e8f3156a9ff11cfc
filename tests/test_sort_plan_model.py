"""The model and generators of test_gpu_sort_plans.py on the CPU: consolidate_np on the sample-defeating and wide-row
generators equals the oracle, its packed-key sort equals np.lexsort, and the plan mirror gives the counts of
sort.cu's plan table."""
import numpy as np
import pytest

import sort_plan_cases as sp
from exact_model import assert_batch_is, consolidate_np, lex_order

N = 300_000


@pytest.mark.parametrize("gen", ["one word", "two words", "wide", "wide, word 0 defeated", "cancelling runs"])
def test_model_equals_oracle(oracle, gen):
    schema, cols, w = {
        "one word": lambda: sp.sample_defeating(N, 1),
        "two words": lambda: sp.sample_defeating(N, 2, two_words=True),
        "wide": lambda: sp.wide_rows(N, 3),
        "wide, word 0 defeated": lambda: sp.wide_rows(N, 4, defeat_word0=True),
        "cancelling runs": lambda: sp.cancelling_runs(N, 20_000, 5),
    }[gen]()
    expect = consolidate_np(schema, cols, w)
    assert_batch_is(oracle.batch_from_columns(schema, cols, w), expect, gen)
    if gen == "cancelling runs":   # one run vanished, the other sums to i64::MIN
        assert not np.any((expect[0][0] == 7) & (expect[0][1] == 9))
        assert expect[1][(expect[0][0] == 1 << 19) & (expect[0][1] == 3)].tolist() == [-(1 << 63)]


def test_sample_defeating_rows_make_equal_splitters():
    """every sampled row is the smallest row, and no other row is"""
    schema, cols, w = sp.sample_defeating(N, 1)
    pos = sp.sample_positions(N)
    assert len(pos) == sp.n_buckets(N) * sp.OVERSAMPLE and np.all(np.diff(pos) > 0) and pos[-1] < N
    smallest = (cols[0] == 0) & (cols[1] == 0)
    assert np.array_equal(np.flatnonzero(smallest), pos)
    schema, cols, w = sp.sample_defeating(N, 1, two_words=True)
    assert sp.KeyPlan(schema, cols, w).W == 2
    assert all(len(np.unique(c[pos])) == 1 for c in cols) and np.array_equal(np.flatnonzero(cols[0] == 0), pos)


def test_lex_order_is_lexsort():
    rng = np.random.default_rng(0)
    for _ in range(200):
        n, L = int(rng.integers(1, 3000)), int(rng.integers(1, 9))
        cols = []
        for _ in range(L):
            b = int(rng.integers(0, 65))
            c = rng.integers(0, 1 << 64, n, dtype=np.uint64, endpoint=False) >> np.uint64(64 - b) if b else np.zeros(n, np.uint64)
            cols.append(rng.choice(c[:3], n) if rng.random() < 0.3 else c)
        assert np.array_equal(lex_order(cols)[0], np.lexsort(cols[::-1])), (n, [int(c.max()).bit_length() for c in cols])


def test_key_plan_mirrors_the_packing():
    schema, cols, w = sp.q7_rows(10_000, 1)
    kp = sp.KeyPlan(schema, cols, w)
    assert kp.W == 2 and kp.bits[3] == 0 and not kp.presorted and not kp.ordered
    kp = sp.KeyPlan(*sp.q7_rows(10_000, 1, run=920))
    assert kp.presorted
    kp = sp.KeyPlan(*sp.wide_rows(10_000, 1))
    assert kp.W == 3 and kp.B == [40, 62, 62]
    assert sp.KeyPlan(*sp.ordered_rows(1000, False, 1)).adoptable
    kp = sp.KeyPlan(*sp.ordered_rows(1000, True, 1))
    assert kp.ordered and not kp.adoptable


@pytest.mark.parametrize("n,name,radix,chunk", [
    (3072, "one chunk", 0, 1),
    (100_000, "top digit", 2, 1),
    (262_144, "splitters(512)", (1 + 5) + 1 + 3, 1),
    (6_291_456, "splitters(8192)", 10, 1),
    (6_291_457, "splitters(16384)", 10, 1),
    (25_165_824, "splitters(32768)", 10, 1),
    (25_165_825, "lsd", 1 + 5, 0),
])
def test_expected_plan_table(n, name, radix, chunk):
    """B = 38 bits, one word: sort.cu's plan table"""
    p = sp.expected_plan(n, 38, 1)
    assert (p.name, p.counts["radix_sort"][0], p.counts["chunk_sort"][0], p.counts["pack_keys"]) == (name, radix, chunk, 1)
    f = sp.expected_plan(n, 38, 1, fallback=True)
    assert f.name == name + " -> lsd fallback"
    assert (f.counts["radix_sort"][0], f.counts["chunk_sort"][0], f.counts["pack_keys"], f.counts["seg_reduce"]) == (radix + 6, chunk, 2, 2)
    if n > sp.CS_HALF:
        assert sp.expected_plan(n, 38, 1, presorted=True).name == "chunks"
    w3 = sp.expected_plan(n, [40, 62, 62], 3)
    assert w3.counts["pack_keys"] == 3 and w3.counts["chunk_sort"][0] == 3 * chunk
