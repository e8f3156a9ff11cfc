"""The long-horizon cases of tests/horizon_cases.py on the CPU oracle, against the non-incremental model."""
import pytest

import horizon_cases as hc


@pytest.mark.parametrize("name", sorted(hc.ALL_CASES))
def test_oracle_horizon(oracle, name):
    hc.ALL_CASES[name](oracle)
