"""The row-shape and view cases of tests/shape_cases.py on the CUDA library: every case against the exact model and
bit for bit against the CPU oracle.  The cases that merge run a second time in child processes with
DBSP_MERGE_NO_TMA=1 (read once per process), where every merge tile is staged row by row with cp.async instead of
TMA bulk copies: at 3 lanes or more only that switch reaches the cp.async path, because the lanes of one allocation
always share a 16-byte phase."""
import os
import subprocess
import sys

import pytest

import shape_cases as sc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(sc.ALL_CASES))
def test_gpu_shapes(cuda, oracle, name):
    sc.ALL_CASES[name](cuda, oracle)


@pytest.mark.parametrize("group", sorted(sc.NO_TMA_GROUPS))
def test_gpu_shapes_no_tma(group):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "shape_cases.py"), group], capture_output=True,
                         text=True, timeout=600, cwd=ROOT, env=dict(os.environ, DBSP_MERGE_NO_TMA="1"))
    tail = out.stdout[-3000:] + out.stderr[-6000:]
    assert out.returncode == 0, tail
    assert f"SHAPES_OK {group} {len(sc.no_tma_cases(group))} cases" in out.stdout, tail
