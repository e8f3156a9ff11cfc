"""Test-only backend: the CPU oracle (oracle/libdbsp_oracle.so) behind the same
C ABI as the product library, with the prefix ``orc_``.  Lives under tests/ on
purpose: the product package cannot reach it."""
import ctypes as C
import os
import subprocess

import numpy as np

import dbsp_b200
from dbsp_b200._capi import CApi
from dbsp_b200.zset import Backend, Batch, Schema

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
ORACLE_LIB = os.path.join(ORACLE_DIR, "libdbsp_oracle.so")


def build_oracle():
    srcs = [os.path.join(ORACLE_DIR, "dbsp_oracle.cpp"), os.path.join(ROOT, "database-stream-processor_b200", "csrc", "validate.h")]
    if not os.path.exists(ORACLE_LIB) or os.path.getmtime(ORACLE_LIB) < max(os.path.getmtime(x) for x in srcs):
        subprocess.check_call(["make", "-C", ORACLE_DIR, "-s"])
    return ORACLE_LIB


class OracleBackend(Backend):
    name = "oracle"

    def __init__(self, lib_path=None):
        """lib_path: another build of the oracle (the sanitizer build of oracle/Makefile) instead of the default one."""
        lib = C.CDLL(lib_path or build_oracle())
        super().__init__(CApi(lib, "orc_"), 0)

    def flat(self, b: Batch):
        """Flat (lanes.., weights) numpy columns of a batch."""
        d = b.download()
        s = b.schema
        if s.nv == 0:
            return [np.asarray(k).view(np.uint64) for k in d["keys"]], d["diffs"]
        counts = np.diff(d["offs"].astype(np.int64))
        keys = [np.repeat(np.asarray(k).view(np.uint64), counts) for k in d["keys"]]
        return keys + [np.asarray(v).view(np.uint64) for v in d["vals"]], d["diffs"]

    def batch_flat_tensors(self, b: Batch, synced: bool = False):
        import torch

        cols, w = self.flat(b)
        return [torch.from_numpy(c.view(np.int64).copy()) for c in cols], torch.from_numpy(w.copy())

    def batch_from_flat_tensors(self, schema: Schema, cols, weights, synced: bool = False) -> Batch:
        return self.batch_from_sorted(schema, [c.numpy().view(np.uint64) for c in cols], weights.numpy(), int(weights.numel()), False)

    def batch_from_device_tensors(self, schema: Schema, cols, weights) -> Batch:
        return self.batch_from_columns(schema, [c.numpy().view(np.uint64) for c in cols], weights.numpy())
