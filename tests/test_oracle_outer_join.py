"""tests/outer_join_cases.py on the CPU oracle with dbsp_antijoin_delta (the row-function build), against the
non-incremental models; and the refusals of the new call and of outer_join."""
import pytest

import outer_join_cases as oc
from rowfn_cases import fn_oracle


@pytest.fixture(scope="module")
def orc():
    return fn_oracle()


@pytest.mark.parametrize("name", sorted(oc.ALL_CASES))
def test_oracle_outer_join(orc, name):
    oc.ALL_CASES[name](orc)


def test_oracle_antijoin_delta_refusals(orc):
    oc.run_refusals(orc)


def test_outer_join_refusals(orc):
    oc.run_python_refusals(orc)


def test_plain_oracle_lacks_antijoin_delta(oracle):
    """The oracle of the dbsp_proj tests has no dbsp_antijoin_delta: its antijoin is the composition, and calling
    the new entry point raises instead of reaching a missing symbol."""
    from dbsp_b200._capi import DbspError

    assert not oracle.api.exports("antijoin_delta")
    with pytest.raises(DbspError, match="orc_antijoin_delta: this library does not export it"):
        oracle.api.call("antijoin_delta", None, None, None, None, None, None)


# The existing antijoin cases, on the library whose Stream.antijoin runs dbsp_antijoin_delta (the dbsp_proj oracle of
# their own test files runs the composition).
def test_golden_antijoin_on_antijoin_delta(orc):
    import golden_cases as gc

    gc.ALL_CASES["antijoin"](orc)


@pytest.mark.parametrize("seed", range(6))
def test_model_antijoin_on_antijoin_delta(orc, seed):
    import test_oracle_model

    test_oracle_model.test_incremental_equals_model(orc, seed)


@pytest.mark.parametrize("name", sorted(n for n in __import__("horizon_cases").ALL_CASES if n.startswith("circuit_")))
def test_horizon_circuit_on_antijoin_delta(orc, name):
    import horizon_cases as hc

    hc.ALL_CASES[name](orc)
