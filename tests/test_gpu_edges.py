"""The integer-domain edge cases of tests/edge_cases.py on the CUDA library: every case against the exact model
and bit for bit against the CPU oracle; plus the join's refusal of a step with 2^32-1 or more matches."""
import numpy as np
import pytest

import edge_cases as ec
from dbsp_b200 import Proj, Schema, Spine, capi, key, lval, rval
from dbsp_b200._capi import DbspError

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(ec.ALL_CASES))
def test_gpu_edges(cuda, oracle, name):
    ec.ALL_CASES[name](cuda, oracle)


def test_join_match_count_overflow(cuda):
    """70 000 x 70 000 rows on one key = 4.9e9 matches: more than the u32 slots of the probe.  The join must refuse
    the step (DBSP_ERR_UNSUPPORTED) without building rows, and the same context must still join correctly.
    Not run on the oracle, which would build the 4.9e9 rows."""
    n = 70_000
    s = Schema("i", "u")
    k = np.full(n, ec.MIN, np.int64).view(np.uint64)
    a = cuda.batch_from_columns(s, [k, np.arange(n, dtype=np.uint64)], np.ones(n, np.int64))
    b = cuda.batch_from_columns(s, [k, np.arange(n, dtype=np.uint64) * np.uint64(3)], np.full(n, 1 << 32, np.int64))
    proj = Proj(Schema("i", "uu"), [key(0), lval(0), rval(0)])
    with pytest.raises(DbspError, match="UNSUPPORTED.*2\\^32-1 or more matches"):
        cuda.join_batches(a, b, proj)
    L = [(ec.MIN, 1, 1 << 32), (ec.MIN, 2, 3), (ec.MAX, 5, -1)]
    R = [(ec.MIN, 7, 1 << 32), (ec.MIN, 8, ec.MIN), (ec.MAX, 9, ec.MIN)]
    out = cuda.join_batches(cuda.batch_from_rows(s, L), cuda.batch_from_rows(s, R), proj)
    ec.em.assert_batch_is(out, ec.em.join(ec.Z(s, L), ec.Z(s, R), proj), "small join after the refusal")
    assert len(out) == 3   # (MIN,1,7) vanishes: 2^32 * 2^32 = 0; (MIN,1,8): 2^32 * MIN = 0 too


@pytest.mark.parametrize("kind", [capi.AGG_MAX, capi.AGG_MIN])
def test_extremum_walk_resolves_extremes(cuda, kind):
    """Max / Min over i64 values at MIN / MAX whose extremes a second batch cancels by wrap (MIN + MIN): every key
    is settled by the walk over the batches' range ends in the order-flipped domain, so the gather fallback (its
    probe kernels) never runs, and the result equals the model's.

    This is the only guard of the walk itself.  A walk that never settles a key (e.g. one that compares candidates
    without the i64 order flip) hands every key to the gather fallback, whose results are right, so the output
    comparisons of every other case still pass.  Hence the check of which kernels ran, by their profiler names
    ("agg_pick" = the walk, "probe_fill" = the gather)."""
    s = Schema("u", "i")
    base = [(k, v, ec.MIN if v in (ec.MIN, ec.MAX) else 1) for k in range(50) for v in ec.I_POOL]
    retract = [(k, v, ec.MIN) for k in range(50) for v in (ec.MIN, ec.MAX)]
    tr, out_tr = Spine(cuda, s), Spine(cuda, s)
    tr.insert(cuda.batch_from_rows(s, base))
    d = cuda.batch_from_rows(s, retract)
    tr.insert(d)
    assert tr.stats()[1] == 2, tr.stats()
    cuda.profile(True)
    out = cuda.aggregate_delta(d, tr, out_tr, kind)
    prof = cuda.profile_read()
    cuda.profile(False)
    zin = ec.Z(s, base + retract)
    ec.em.assert_batch_is(out, ec.em.aggregate_delta(ec.Z(s, retract), zin, ec.Z(s), kind), "walk at the extremes")
    assert "agg_pick" in prof and "probe_fill" not in prof, sorted(prof)
