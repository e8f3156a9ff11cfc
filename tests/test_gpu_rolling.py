"""tests/rolling_cases.py on the CUDA library: every case against the non-incremental model and bit for bit against
the CPU oracle at every step; the refusals, with the oracle's texts; the `rolling` profile class; and Nexmark
rolling_bids, plain and watermark forms, at 5 M events per step over 5 steps, equal to the oracle's output at every
step."""
import pytest

import rolling_cases as rc
from dbsp_b200 import Before, Max, RelRange, RootCircuit, Schema
from rowfn_cases import fn_oracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def orc():
    return fn_oracle()


@pytest.mark.parametrize("name", sorted(rc.ALL_CASES))
def test_gpu_rolling(cuda, orc, name):
    rc.ALL_CASES[name](cuda, orc)


def test_gpu_rolling_refusals(cuda, orc):
    """one refusal per rule, with the same status and text as the oracle's"""
    assert rc.run_refusals(cuda) == rc.run_refusals(orc)


def test_gpu_rolling_profile_class(cuda):
    c = RootCircuit(cuda)
    s, h = c.add_input_indexed_zset(Schema("u", "ui"))
    s.partitioned_rolling_aggregate(Max, RelRange(Before(10), Before(0)))
    h.append([(i % 7, i, i, 1) for i in range(1000)])
    cuda.profile(True)
    c.step()
    prof = cuda.profile_read()
    cuda.profile(False)
    # the first step (an empty output trace) times five scopes: the intervals, the range search and the copy of the
    # input gather, the sparse table's levels, and the outputs
    assert prof["rolling"]["launches"] == 5 and prof["rolling"]["alg_bytes"] > 0


@pytest.mark.parametrize("watermark", [False, True], ids=["plain", "watermark"])
def test_gpu_rolling_bids_scale(cuda, orc, watermark):
    """Nexmark rolling_bids at 5 M events per step for 5 steps: both outputs of every step bit-identical between the
    CUDA library and the oracle"""
    rc.run_bids_pair(cuda, orc, watermark)
