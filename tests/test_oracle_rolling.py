"""tests/rolling_cases.py on the CPU oracle with dbsp_rolling_aggregate (the row-function build), against the
non-incremental model, and the refusals of valid_rolling."""
import pytest

import rolling_cases as rc
from rowfn_cases import fn_oracle


@pytest.fixture(scope="module")
def orc():
    return fn_oracle()


@pytest.mark.parametrize("name", sorted(rc.ALL_CASES))
def test_oracle_rolling(orc, name):
    rc.ALL_CASES[name](orc)


def test_oracle_rolling_refusals(orc):
    rc.run_refusals(orc)


def test_plain_oracle_lacks_rolling(oracle):
    from dbsp_b200 import Before, Max, RelRange, RootCircuit, Schema
    from dbsp_b200._capi import DbspError

    c = RootCircuit(oracle)
    s, _ = c.add_input_indexed_zset(Schema("u", "ui"))
    with pytest.raises(DbspError, match="rolling_aggregate"):
        s.partitioned_rolling_aggregate(Max, RelRange(Before(1), Before(0)))
