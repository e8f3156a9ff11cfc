"""tests/upsert_cases.py on the CPU oracle with dbsp_upsert_commands / dbsp_upsert_delta (the row-function build),
against the non-incremental model: the reference's literals, command order, shapes, trace states, weights other than
1, a save / load of the table trace, and the refusals."""
import pytest

import upsert_cases as uc
from rowfn_cases import fn_oracle


@pytest.fixture(scope="module")
def orc():
    return fn_oracle()


@pytest.mark.parametrize("name", sorted(uc.ALL_CASES))
def test_oracle_upsert(orc, name):
    uc.ALL_CASES[name](orc)


def test_oracle_upsert_save_load(orc, tmp_path):
    uc.run_save_load(orc, tmp_path)


def test_oracle_upsert_refusals(orc):
    uc.run_refusals(orc)


def test_upsert_python_refusals(orc):
    uc.run_python_refusals(orc)


def test_plain_oracle_lacks_upsert(oracle):
    uc.run_plain_oracle_lacks(oracle)
