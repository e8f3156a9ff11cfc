"""tests/fold_cases.py on the CUDA library: every case against the non-incremental model and bit for bit against the
CPU oracle with dbsp_aggregate_fold; the refusals of the new call; its profile class; and Nexmark q18 / q6, on the
reference's test data and at 5 M events per step against the oracle."""
import pytest

import fold_cases as fc
from rowfn_cases import fn_oracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def orc():
    return fn_oracle()


@pytest.mark.parametrize("name", sorted(fc.ALL_CASES))
def test_gpu_fold(cuda, orc, name):
    fc.ALL_CASES[name](cuda, orc)


def test_gpu_aggregate_fold_refusals(cuda):
    fc.run_refusals(cuda)


def test_gpu_fold_python_refusals(cuda):
    fc.run_python_refusals(cuda)


def test_gpu_agg_fold_profile_class(cuda):
    """k_agg_fold is timed under its own name, with G's rows and the affected keys' output lanes as its bytes."""
    fc.run_profile_class(cuda)


@pytest.mark.parametrize("query", ["q18", "q6"])
def test_gpu_fold_golden(cuda, query):
    fc.run_golden(cuda, query)


@pytest.mark.parametrize("query", ["q18", "q6"])
def test_gpu_fold_generated(cuda, query):
    fc.run_generated(cuda, query)


@pytest.mark.parametrize("query", ["q18", "q6"])
def test_gpu_fold_nexmark(cuda, orc, query):
    """5 M events per step for 5 steps, every step's output equal to the oracle's."""
    fc.run_nexmark_pair(cuda, orc, query, n_events=5_000_000, steps=5)
