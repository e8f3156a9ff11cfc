"""The long-horizon cases of tests/horizon_cases.py on the CUDA library: every step against the non-incremental model
and bit for bit against the CPU oracle, the traces' layers at every checkpoint against the schedule model
(horizon_cases.SpineModel), and the kernel paths each regime is for asserted from the profiler's kernel names."""
import pytest

import horizon_cases as hc

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(hc.ALL_CASES))
def test_gpu_horizon(cuda, oracle, name):
    hc.ALL_CASES[name](cuda, oracle)
