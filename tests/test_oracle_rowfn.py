"""Row functions (tests/rowfn_cases.py) on the CPU oracle, against the model of rowfn_cases.py."""
import pytest

import rowfn_cases as rc


@pytest.fixture(scope="module")
def oracle():
    """The CPU oracle with the row-function entry points."""
    return rc.fn_oracle()


def test_oracle_rowfn_every_op(oracle):
    rc.run_every_op(oracle)


def test_oracle_rowfn_tables(oracle):
    rc.run_tables(oracle)


def test_oracle_rowfn_map_join_weigh(oracle):
    rc.run_map_join_weigh(oracle)


def test_oracle_rowfn_sizes(oracle):
    rc.run_sizes(oracle)


def test_oracle_rowfn_random_programs(oracle):
    rc.run_random_programs(oracle)


@pytest.mark.parametrize("query", ["q0", "q3", "q4", "q7"])
def test_oracle_rowfn_lowering(oracle, query):
    rc.run_lowering(oracle, query)


def test_oracle_rowfn_refusals(oracle):
    rc.run_refusals(oracle)


def test_oracle_reference_q1_q2(oracle):
    rc.run_reference_q1_q2(oracle)


@pytest.mark.parametrize("name", sorted(rc.ABS_CASES))
def test_oracle_filter_map_abs(oracle, name):
    rc.run_abs_case(oracle, name)


def test_dbsp_proj_bytes_unchanged():
    rc.run_dbsp_proj_bytes_unchanged()


def test_oracle_without_row_functions_refuses_them():
    """The oracle of the dbsp_proj tests exports no row functions: its backend binds every other call and a row
    function raises instead of running."""
    import numpy as np
    from dbsp_b200 import Proj, Schema, col
    from dbsp_b200._capi import DbspError
    from oracle_backend import OracleBackend

    be = OracleBackend()
    p = Proj(Schema("u"), [col(0) % 7])
    with pytest.raises(DbspError, match="orc_batch_from_table_fn: this library has no row functions"):
        be.batch_from_table([np.arange(4, dtype=np.uint64)], p)
    assert len(be.batch_from_table([np.arange(4, dtype=np.uint64)], Proj(Schema("u"), [col(0)]))) == 4
