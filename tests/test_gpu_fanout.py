"""Fan-outs (tests/fanout_cases.py) on the CUDA library: every case against the model and, bit for bit, the
row-function oracle; Nexmark q5_hop at 5 M events per step."""
import pytest

import fanout_cases as fc
from parity_util import run_nexmark_pair

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def oracle():
    """The CPU oracle with the row-function and fan-out entry points."""
    return fc.fn_oracle()


def test_cuda_fanout_n_outs(cuda, oracle):
    fc.run_n_outs(cuda, oracle)


def test_cuda_fanout_entry_points(cuda, oracle):
    fc.run_entry_points(cuda, oracle)


def test_cuda_fanout_random_programs(cuda, oracle):
    fc.run_random_programs(cuda, oracle, n_programs=150)


def test_cuda_fanout_shard_data(cuda):
    fc.run_shard_data(cuda)


def test_cuda_fanout_one_is_the_plain_closure(cuda):
    fc.run_fanout_one(cuda)


def test_cuda_fanout_refusals(cuda, oracle):
    fc.run_refusals(cuda, oracle)
    cuda.sync()


def test_cuda_q5_hop(cuda):
    fc.run_q5_hop(cuda)


def test_cuda_nexmark_q5_hop_5m(cuda, oracle):
    """5 steps of 5 M events: every step's output equal to the oracle's."""
    assert run_nexmark_pair(cuda, oracle, "q5_hop", n_events=25_000_000, step=5_000_000) > 0
