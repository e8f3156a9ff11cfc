"""The row-shape and view cases of tests/shape_cases.py on the CPU oracle, against the exact model."""
import pytest

import shape_cases as sc


@pytest.mark.parametrize("name", sorted(sc.ALL_CASES))
def test_oracle_shapes(oracle, name):
    sc.ALL_CASES[name](oracle)
