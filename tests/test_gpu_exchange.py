"""The in-library exchange (csrc/comm.cu) on one GPU: P contexts of one process, one thread per rank, checked against
the exact model of tests/exchange_model.py (see tests/exchange_worker.py for the scenarios and the harness's rules).

Each (scenario, P) runs in its own process, because the environment the ranks need must be set before CUDA starts,
and this process already holds a context:
  * CUDA_DEVICE_MAX_CONNECTIONS=32: every context's stream gets its own hardware queue, so that no rank's signal
    kernel waits behind another rank's spinning wait kernel;
  * DBSP_COMM_TIMEOUT_S=20: a protocol bug ends the round with an error status instead of a long wait;
  * DBSP_POOL_SLAB_MB=256: P pools of 256 MiB slabs instead of 8 GiB each;
  * CUDA_MODULE_LOADING=EAGER: ranks that share a device share one CUDA context, and under lazy loading a rank's
    first launch of a kernel waits for a peer's spinning wait kernel (dbsp_comm_connect refuses that setup).
The cross-process CUDA IPC mapping and the NVLink transport stay with tests/test_multigpu.py (>= 2 GPUs)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "exchange_worker.py")

pytestmark = pytest.mark.gpu

SCENARIOS = ["allreduce", "shard_model", "sizes", "receiver_paths", "cancel_across_ranks", "gather", "shard2",
             "retention", "slot_overflow", "circuits"]
AT_32 = ["allreduce", "shard_model", "gather"]   # DBSP_COMM_MAX_RANKS: one warp polls 32 peers
CASES = [(s, P) for s in SCENARIOS for P in (2, 3, 4, 8)] + [(s, 32) for s in AT_32]
ENV = {"CUDA_DEVICE_MAX_CONNECTIONS": "32", "DBSP_COMM_TIMEOUT_S": "20", "DBSP_POOL_SLAB_MB": "256",
       "CUDA_MODULE_LOADING": "EAGER"}


@pytest.mark.skipif(os.environ.get("CUDA_LAUNCH_BLOCKING", "0") not in ("", "0"),
                    reason="CUDA_LAUNCH_BLOCKING serialises the ranks' streams: one rank's wait kernel would block "
                           "the signal kernels of its peers")
@pytest.mark.parametrize("scenario,P", CASES, ids=[f"{s}-P{P}" for s, P in CASES])
def test_exchange_one_gpu(scenario, P):
    out = subprocess.run([sys.executable, WORKER, scenario, str(P)], capture_output=True, text=True, timeout=300,
                         cwd=ROOT, env=dict(os.environ, **ENV))
    tail = out.stdout[-3000:] + out.stderr[-6000:]
    assert out.returncode == 0, tail
    assert f"EXCHANGE_OK {scenario} P={P}" in out.stdout, tail


def test_shared_device_needs_eager_loading():
    """Under lazy kernel loading, two ranks on one device are refused at dbsp_comm_connect, before any round."""
    code = ("import sys; sys.path.insert(0, 'tests'); import exchange_worker as xw\n"
            "try:\n    xw.Group(2, 1 << 20)\nexcept xw.DbspError as e:\n    print('REFUSED', e)\n")
    env = dict(os.environ, **ENV)
    env["CUDA_MODULE_LOADING"] = "LAZY"
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120, cwd=ROOT, env=env)
    assert "REFUSED" in out.stdout and "UNSUPPORTED" in out.stdout and "CUDA_MODULE_LOADING=EAGER" in out.stdout, (
        out.stdout[-2000:] + out.stderr[-2000:])
