"""tests/fold_cases.py on the CPU oracle with dbsp_aggregate_fold (the row-function build), against the
non-incremental model; the refusals of the new call and of Fold; and Nexmark q18 / q6 on the reference's own test
data and on generated events against GROUP BY models."""
import pytest

import fold_cases as fc
from rowfn_cases import fn_oracle


@pytest.fixture(scope="module")
def orc():
    return fn_oracle()


@pytest.mark.parametrize("name", sorted(fc.ALL_CASES))
def test_oracle_fold(orc, name):
    fc.ALL_CASES[name](orc)


def test_oracle_aggregate_fold_refusals(orc):
    fc.run_refusals(orc)


def test_fold_python_refusals(orc):
    fc.run_python_refusals(orc)


def test_plain_oracle_lacks_aggregate_fold(oracle):
    fc.run_plain_oracle_lacks(oracle)


@pytest.mark.parametrize("query", ["q18", "q6"])
def test_oracle_fold_golden(orc, query):
    fc.run_golden(orc, query)


@pytest.mark.parametrize("query", ["q18", "q6"])
def test_oracle_fold_generated(orc, query):
    fc.run_generated(orc, query)
