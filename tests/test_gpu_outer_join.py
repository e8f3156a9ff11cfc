"""tests/outer_join_cases.py on the CUDA library: every case against the non-incremental models and bit for bit
against the CPU oracle with dbsp_antijoin_delta; the refusals of the new call; and the skewed key, which the
composition the antijoin replaced refuses."""
import pytest

import outer_join_cases as oc
from rowfn_cases import fn_oracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def orc():
    return fn_oracle()


@pytest.mark.parametrize("name", sorted(oc.ALL_CASES))
def test_gpu_outer_join(cuda, orc, name):
    oc.ALL_CASES[name](cuda, orc)


def test_gpu_antijoin_delta_refusals(cuda):
    oc.run_refusals(cuda)


def test_gpu_skew_composition_refused(cuda):
    oc.run_skew_composition_refused(cuda)


def test_gpu_antijoin_profile_class(cuda):
    """The new kernel is timed under its own name, with its algorithmic bytes (28 per delta row)."""
    oc.run_profile_class(cuda)


def test_gpu_q17_first5_nexmark(cuda, orc):
    """q17's first five outer joins at 5 M events per step for 5 steps, equal to the oracle at every step."""
    oc.run_q17_nexmark(cuda, orc, n_events=5_000_000, steps=5)
