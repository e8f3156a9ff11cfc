"""The CUDA library and the CPU oracles refuse alike: every refusal runner of the suite runs on the CUDA library and on
its oracle with each refusal recorded as (call, status, text), and the two sequences are byte-identical.  Calls only
the CUDA library serves are dropped by name.  The two-fault cases of tests/check_order_cases.py run here too."""
import pytest

import check_order_cases as cc
import fanout_cases
import fold_cases
import outer_join_cases
import refusal_cases
import rowfn_cases
import upsert_cases
from rowfn_cases import fn_oracle

pytestmark = pytest.mark.gpu

# asynchronous reads, device columns, the profile and the exchange protocol: the oracle is one worker without a device
CUDA_ONLY = {"batch_download_begin", "batch_device_columns", "ctx_profile", "ctx_profile_read", "comm_connect", "shard", "gather"}
# the modules whose runners check their refusals with refusal_cases.refused, imported by name
MODULES = (refusal_cases, rowfn_cases, fanout_cases, fold_cases, outer_join_cases)
UPSERT_CALLS = ("upsert_commands", "upsert_delta")   # upsert_cases checks them with a helper of its own


@pytest.fixture(scope="module")
def orc_fn():
    return fn_oracle()


def recorded(monkeypatch, runner, be):
    """The (call, status, text) of every refusal `runner(be)` checks, in order, each still asserted as before."""
    log = []
    checked = refusal_cases.refused

    def record(b, call, *args, **kw):
        msg = checked(b, call, *args, **kw)
        log.append((call, kw.get("status", refusal_cases.INVALID), msg))
        return msg

    with monkeypatch.context() as m:
        for mod in MODULES:
            m.setattr(mod, "refused", record)
        for call in UPSERT_CALLS:
            def raw(*args, fn=getattr(be.api, "_" + call), call=call):
                rc = fn(*args)
                if rc:
                    log.append((call, rc, be.api._last_error().decode()))
                return rc
            m.setattr(be.api, "_" + call, raw)
        runner(be)
    assert log, "the runner checked no refusal"
    return [r for r in log if r[0] not in CUDA_ONLY]


def assert_same_refusals(monkeypatch, runner, cuda, ref):
    got, want = recorded(monkeypatch, runner, cuda), recorded(monkeypatch, runner, ref)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"refusal {i}: CUDA {g!r}, oracle {w!r}"
    assert len(got) == len(want), f"{len(got)} refusals on CUDA, {len(want)} on the oracle"


@pytest.mark.parametrize("group", sorted(refusal_cases.GROUPS))
def test_refusal_texts_match_oracle(monkeypatch, cuda, oracle, group):
    assert_same_refusals(monkeypatch, refusal_cases.GROUPS[group], cuda, oracle)
    cuda.sync()


@pytest.mark.parametrize("module", [rowfn_cases, fanout_cases, fold_cases, upsert_cases, outer_join_cases],
                         ids=lambda m: m.__name__)
def test_rowfn_refusal_texts_match_oracle(monkeypatch, cuda, orc_fn, module):
    assert_same_refusals(monkeypatch, module.run_refusals, cuda, orc_fn)
    cuda.sync()


@pytest.mark.parametrize("case", sorted(cc.CASES))
def test_cuda_check_order(cuda, case):
    cc.CASES[case](cuda)
    cuda.sync()
