"""Two faults at once (tests/check_order_cases.py) on both CPU oracles: the rule first in the call's audit row wins,
with the CUDA library's status and text.  The plain oracle skips the calls it does not export.  DBSP_ORACLE_LIB
selects another build of the plain oracle, as in tests/test_oracle_refusals.py (the sanitizer build)."""
import os

import pytest

import check_order_cases as cc
from rowfn_cases import fn_oracle


@pytest.fixture(scope="module")
def be(oracle):
    path = os.environ.get("DBSP_ORACLE_LIB")
    if not path:
        return oracle
    from oracle_backend import OracleBackend

    return OracleBackend(path)


@pytest.fixture(scope="module")
def orc_fn():
    return fn_oracle()


@pytest.mark.parametrize("case", sorted(cc.CASES))
def test_oracle_check_order(be, case):
    cc.CASES[case](be)


@pytest.mark.parametrize("case", sorted(cc.CASES))
def test_oracle_fn_check_order(orc_fn, case):
    cc.CASES[case](orc_fn)
