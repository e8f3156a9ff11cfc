"""The C-ABI library loads and exports every symbol include/dbsp_b200.h declares
(no compute calls: this runs without a GPU)."""
import ctypes
import os
import re

import dbsp_b200
from dbsp_b200._capi import CApi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "dbsp_b200.h")).read()
    return sorted(set(re.findall(r"\b(dbsp_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported():
    import __graft_entry__ as ge

    ge.build()
    lib = ctypes.CDLL(ge.LIB)
    syms = header_symbols()
    assert len(syms) >= 35
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in the header but not exported"
    # and the Python binding covers every one of them
    assert sorted(CApi.symbols("dbsp_")) == syms


def test_no_cpu_fallback():
    """Without a device the product backend must fail loudly, not fall back."""
    import pytest
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from dbsp_b200.runtime import Runtime
    from dbsp_b200._capi import DbspError

    with pytest.raises(DbspError, match="NO_DEVICE"):
        Runtime(0)


# ---- the error contract, as far as it needs no device (tests/refusal_cases.py has the rest) ------------------------
def _api():
    import __graft_entry__ as ge

    ge.build()
    return CApi(ctypes.CDLL(ge.LIB), "dbsp_")


def test_null_context_is_refused_without_a_device():
    """A NULL context comes back as DBSP_ERR_INVALID with a text naming the call and `ctx`; nothing is dereferenced."""
    api = _api()
    out, n = ctypes.c_void_p(), ctypes.c_uint64()
    calls = {
        "ctx_sync": (None,), "ctx_stats": (None, None, None, None, 0), "ctx_sync_stats": (None, None, None, 0), "ctx_profile": (None, 1),
        "batch_empty": (None, None, ctypes.byref(out)), "batch_neg": (None, None, ctypes.byref(out)), "batcher_new": (None, None, ctypes.byref(out)),
        "spine_new": (None, None, ctypes.byref(out)), "spine_load": (None, b"unused", ctypes.byref(out)), "map_index": (None, None, None, ctypes.byref(out)),
        "shard": (None, None, ctypes.byref(out)), "comm_info": (None, None, None, None), "comm_destroy": (None,), "allreduce_max_u64": (None, ctypes.byref(n)),
    }
    for name, args in calls.items():
        assert getattr(api, "_" + name)(*args) == 1, name
        msg = api._last_error().decode()
        assert name in msg and "ctx is NULL" in msg, (name, msg)
        assert not out.value
    assert api._ctx_stream(None) is None
    assert api._ctx_destroy(None) == 0
    assert api._ctx_create(0, None) == 1 and "out is NULL" in api._last_error().decode()
    assert api._ctx_create(-1, ctypes.byref(out)) == 1 and "device" in api._last_error().decode() and not out.value


def test_handle_calls_without_a_context():
    """Calls that take no context refuse NULL handles and out-pointers; every *_free is a no-op on NULL."""
    api = _api()
    n = ctypes.c_uint64()
    for name, args, arg in (("batch_len", (None, ctypes.byref(n)), "batch"), ("batch_schema", (None, None), "batch"),
                            ("batch_clone", (None, None), "batch"), ("batch_device_columns", (None, None, None), "batch"),
                            ("batcher_tuples", (None, ctypes.byref(n)), "batcher"), ("spine_len", (None, ctypes.byref(n), None), "spine")):
        assert getattr(api, "_" + name)(*args) == 1, name
        msg = api._last_error().decode()
        assert name in msg and f"{arg} is NULL" in msg, (name, msg)
    for name in ("batch_free", "spine_free", "merger_free", "batcher_free", "upload_free", "download_finish"):
        assert getattr(api, "_" + name)(None) == 0, name


def test_proj_table_mask_needs_no_device():
    from dbsp_b200 import Proj, Schema, const, key, lval, rval
    from dbsp_b200._capi import CProj

    api = _api()
    p = Proj(Schema("u", "uu"), [lval(7), key(2) + rval(4), const(9)], where=[lval(0).lt(const(3)), const(1).eq(key(5))])
    assert api._proj_table_mask(p.c()) == (1 << 7) | (1 << 2) | (1 << 4) | (1 << 0) | (1 << 5)
    assert api._proj_table_mask(Proj(Schema("u"), [const(1)]).c()) == 0
    assert api._proj_table_mask(Proj(Schema("u"), [-lval(3)]).c()) == 1 << 3   # the unused second operand of NEG names no column
    # what no table can satisfy reads no column: a NULL projection, a column past the eighth, a malformed struct
    assert api._proj_table_mask(None) == 0
    assert api._proj_table_mask(Proj(Schema("u"), [lval(8)]).c()) == 0
    bad = CProj.from_buffer_copy(p._c)
    bad.n_pred = 200
    assert api._proj_table_mask(ctypes.byref(bad)) == 0


def audit_symbols():
    """The symbols of the argument audit in DESIGN.md §1 (one table row per entry point: `| \\`dbsp_x\\` | ...`)."""
    src = open(os.path.join(ROOT, "DESIGN.md")).read()
    start = src.index("### Error contract")
    end = src.index("\n## ", start)
    return sorted(re.findall(r"^\| `(dbsp_[a-z0-9_]+)` \|", src[start:end], re.M))


def test_every_entry_point_is_in_the_argument_audit():
    """A new entry point cannot skip the audit of its arguments: the table lists exactly the header's symbols."""
    assert audit_symbols() == header_symbols()
