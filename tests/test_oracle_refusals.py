"""The ABI's error contract (tests/refusal_cases.py) on the CPU oracle, which sits behind the same ABI with the same
validators: a check that is missing shows here as a failed assertion or as a crash of a CPU process.
DBSP_ORACLE_LIB selects another build of the oracle — the sanitizer build of oracle/Makefile (`make -C oracle sanitize`,
run with the sanitizer runtime preloaded), under which an overrun is reported instead of survived."""
import os

import pytest

import refusal_cases as rc


@pytest.fixture(scope="module")
def be(oracle):
    path = os.environ.get("DBSP_ORACLE_LIB")
    if not path:
        return oracle
    from oracle_backend import OracleBackend

    return OracleBackend(path)


@pytest.mark.parametrize("group", sorted(rc.GROUPS))
def test_oracle_refusals(be, group):
    rc.GROUPS[group](be)


def test_oracle_snapshot_refusals(be, tmp_path):
    rc.run_snapshot_refusals(be, tmp_path)


def test_oracle_snapshot_accepts(be, tmp_path):
    rc.run_snapshot_accepts(be, tmp_path)


def test_snapshot_writer_round_trips():
    """The test's own reader / writer of the snapshot format, on a file it builds itself."""
    bt = {"present": 1, "n": 2, "lanes": [[1, 2], [5, 4]], "w": [1, -1]}
    none = {"present": 0, "n": 0, "lanes": [], "w": []}
    snap = {"magic": rc.MAGIC, "nk": 1, "nv": 1, "types": [0, 1] + [0] * 6, "has_bound": 1, "has_vbound": 0, "effort": 1, "n_layers": 2,
            "bound": [3] + [0] * 7, "vbound": [0] * 8,
            "layers": [{"kind": 0, "remaining": 0, "batches": [none, none]}, {"kind": 2, "remaining": 4, "batches": [bt, bt]}]}
    data = rc.write_snapshot(snap)
    back, cuts, mids = rc.parse_snapshot(data)
    assert back == snap and cuts[-1][0] == len(data) and len(mids) == 6
