"""Row functions (tests/rowfn_cases.py) on the CUDA library: every case against the model and, bit for bit, the
oracle; Nexmark q1 and q2 at 5 M events per step."""
import pytest

import rowfn_cases as rc
from parity_util import run_nexmark_pair

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def oracle():
    """The CPU oracle with the row-function entry points."""
    return rc.fn_oracle()


def test_cuda_rowfn_every_op(cuda, oracle):
    rc.run_every_op(cuda, oracle)


def test_cuda_rowfn_tables(cuda, oracle):
    rc.run_tables(cuda, oracle)


def test_cuda_rowfn_map_join_weigh(cuda, oracle):
    rc.run_map_join_weigh(cuda, oracle)


def test_cuda_rowfn_sizes(cuda, oracle):
    rc.run_sizes(cuda, oracle)


def test_cuda_rowfn_random_programs(cuda, oracle):
    rc.run_random_programs(cuda, oracle, n_programs=200)


@pytest.mark.parametrize("query", ["q0", "q3", "q4", "q7"])
def test_cuda_rowfn_lowering(cuda, query):
    rc.run_lowering(cuda, query)


def test_cuda_rowfn_refusals(cuda, oracle):
    rc.run_refusals(cuda, oracle)
    cuda.sync()


def test_cuda_reference_q1_q2(cuda):
    rc.run_reference_q1_q2(cuda)


@pytest.mark.parametrize("name", sorted(rc.ABS_CASES))
def test_cuda_filter_map_abs(cuda, name):
    rc.run_abs_case(cuda, name)


@pytest.mark.parametrize("query", ["q1", "q2"])
def test_cuda_nexmark_q1_q2_5m(cuda, oracle, query):
    """5 steps of 5 M events: every step's output equal to the oracle's."""
    assert run_nexmark_pair(cuda, oracle, query, n_events=25_000_000, step=5_000_000) > 0
