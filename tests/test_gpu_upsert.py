"""tests/upsert_cases.py on the CUDA library: every case against the non-incremental model and bit for bit against the
CPU oracle; the refusals; the `upsert` profile class; and 5 M commands per step into a map of 20 M live keys, equal
to the oracle's output at every step."""
import numpy as np
import pytest

import upsert_cases as uc
from dbsp_b200 import Schema, Spine
from rowfn_cases import fn_oracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def orc():
    return fn_oracle()


@pytest.mark.parametrize("name", sorted(uc.ALL_CASES))
def test_gpu_upsert(cuda, orc, name):
    uc.ALL_CASES[name](cuda, orc)


def test_gpu_upsert_save_load(cuda, tmp_path):
    uc.run_save_load(cuda, tmp_path)


def test_gpu_upsert_refusals(cuda):
    uc.run_refusals(cuda)


def test_gpu_upsert_python_refusals(cuda):
    uc.run_python_refusals(cuda)


def test_gpu_upsert_profile_class(cuda):
    """k_upsert_last is timed under `upsert`, with the key and command lanes read and two flag arrays written."""
    s = Schema("uu", "u")
    n = 10_000
    k = np.arange(n, dtype=np.uint64) % 977
    cmds = cuda.upsert_commands(s, [k, k, k])
    cuda.profile(True)
    cuda.upsert_delta(cmds, Spine(cuda, s))
    prof = cuda.profile_read()
    cuda.profile(False)
    assert prof["upsert"]["launches"] == 1
    assert prof["upsert"]["alg_bytes"] == n * 3 * 8 + (n + 1) * 8


def test_gpu_upsert_scale(cuda, orc):
    uc.run_scale(cuda, orc)
