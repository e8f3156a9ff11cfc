"""The ABI's error contract (tests/refusal_cases.py) on the CUDA library: every refusal comes back from the host
with nothing launched, copied or waited for, and every accepted twin matches the exact model and, bit for bit, the
oracle."""
import pytest

import refusal_cases as rc

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("group", sorted(rc.GROUPS))
def test_cuda_refusals(cuda, oracle, group):
    rc.GROUPS[group](cuda, oracle)
    cuda.sync()


def test_cuda_snapshot_refusals(cuda, oracle, tmp_path):
    """Files written by the CUDA library, damaged, and refused by both libraries for the same reason."""
    rc.run_snapshot_refusals(cuda, tmp_path, oracle)
    cuda.sync()


def test_cuda_snapshot_accepts(cuda, oracle, tmp_path):
    rc.run_snapshot_accepts(cuda, tmp_path, oracle)


def test_oracle_snapshots_refused_alike(cuda, oracle, tmp_path):
    """The other direction: files written by the oracle, damaged, and refused by the CUDA library alike."""
    rc.run_snapshot_refusals(oracle, tmp_path, cuda)
    cuda.sync()
