"""The integer-domain edge cases of tests/edge_cases.py on the CPU oracle, against the exact model."""
import pytest

import edge_cases as ec


@pytest.mark.parametrize("name", sorted(ec.ALL_CASES))
def test_oracle_edges(oracle, name):
    ec.ALL_CASES[name](oracle)
