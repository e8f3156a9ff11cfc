"""Fan-outs (tests/fanout_cases.py) on the row-function CPU oracle, against the model of fanout_cases.py."""
import pytest

import fanout_cases as fc


@pytest.fixture(scope="module")
def oracle():
    """The CPU oracle with the row-function and fan-out entry points."""
    return fc.fn_oracle()


def test_oracle_fanout_n_outs(oracle):
    fc.run_n_outs(oracle)


def test_oracle_fanout_entry_points(oracle):
    fc.run_entry_points(oracle)


def test_oracle_fanout_random_programs(oracle):
    fc.run_random_programs(oracle)


def test_oracle_fanout_shard_data(oracle):
    fc.run_shard_data(oracle)


def test_oracle_fanout_one_is_the_plain_closure(oracle):
    fc.run_fanout_one(oracle)


def test_oracle_fanout_refusals(oracle):
    fc.run_refusals(oracle)


def test_oracle_q5_hop(oracle):
    fc.run_q5_hop(oracle)


def test_fanout_closures_stay_in_flat_map():
    """A fan-out closure is refused by the calls that take one row per input row, before anything runs."""
    from dbsp_b200 import Proj, Schema, fanout_index, key
    from dbsp_b200.zset import _factor, _fn

    p = Proj(Schema("u"), [key(0) + fanout_index()], fanout=2)
    for call in ("join_batches", "join_delta_trace"):
        with pytest.raises(ValueError, match="fan-out"):
            _fn(call, p)
    with pytest.raises(ValueError, match="fan-out"):
        _factor(p)


def test_oracle_without_row_functions_refuses_fanouts():
    """The oracle of the dbsp_proj tests exports no fan-out: calling one raises instead of running."""
    import numpy as np
    from dbsp_b200 import Proj, Schema, col, fanout_index
    from dbsp_b200._capi import DbspError
    from oracle_backend import OracleBackend

    be = OracleBackend()
    p = Proj(Schema("u"), [col(0) + fanout_index()], fanout=2)
    with pytest.raises(DbspError, match="orc_batch_from_table_fanout: this library has no row functions"):
        be.batch_from_table([np.arange(4, dtype=np.uint64)], p)
    with pytest.raises(DbspError, match="orc_fanout_table_mask"):
        be.proj_table_mask(p)
