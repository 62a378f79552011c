"""The job entry point with TAD_STREAM_INPUT=1 TAD_DEVICE_TEXT=1 on the real engine: main() over a 2M-row ClickHouse
double in 65,536-row blocks, the address text dictionary-encoded on the GPU, against the default one-shot path, with no
budget, with a device budget that forces hash-range passes and with the same budget plus a host row store."""
import numpy as np
import pytest

from theia_b200 import anomaly_detection as ad

from .test_gpu_job_entry_stream import BLOCK, HOST, _Recording, canonical_rows, same
from .test_gpu_stream import BUDGET_4
from .test_job_entry_stream import TableTransport, make_table

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    """A context of its own: the budgets set here must not reach the session's engine."""
    from theia_b200.engine import TadEngine
    e = TadEngine(device=0)
    yield e
    e.close()


@pytest.mark.parametrize("dual_stack", [False, True])
def test_device_text_entry_equals_the_one_shot_entry(eng, dual_stack, monkeypatch):
    table = make_table(series=20000, points=100, seed=84, dual_stack=dual_stack, block_rows=BLOCK)     # 2M rows
    argv = ["--algo", "EWMA", "--id", "gpu-text"]
    for v in ("TAD_STREAM_INPUT", "TAD_HOST_BUDGET", "TAD_DEVICE_TEXT", "TAD_IPV4_PUSHDOWN"):
        monkeypatch.delenv(v, raising=False)
    eng.set_memory_budget(0)
    eng.set_host_budget(0)
    tr = TableTransport(table, block_rows=BLOCK)
    assert ad.main(argv, engine=eng, transport=tr) == 0
    want = canonical_rows(tr.inserts[0][1])
    assert len(want["id"]) > 1
    if dual_stack:
        assert any(":" in s for s in want["sourceIP"])
    monkeypatch.setenv("TAD_STREAM_INPUT", "1")
    monkeypatch.setenv("TAD_DEVICE_TEXT", "1")
    try:
        for budget, host in ((0, None), (BUDGET_4, None), (BUDGET_4, HOST)):
            eng.set_memory_budget(budget)
            if host is None:
                monkeypatch.delenv("TAD_HOST_BUDGET", raising=False)
                eng.set_host_budget(0)
            else:
                monkeypatch.setenv("TAD_HOST_BUDGET", str(host))
            rec, tr = _Recording(eng), TableTransport(table, block_rows=BLOCK)
            assert ad.main(argv, engine=rec, transport=tr) == 0
            what = (dual_stack, budget, host)
            assert same(canonical_rows(tr.inserts[0][1]), want), what
            (mem,) = rec.memory
            if budget:
                assert mem["passes"] >= 4 and mem["peak_workspace_bytes"] <= budget, (what, mem)
            if host:
                assert mem["stored_rows"] > 0 and len(tr.selects) == 1, (what, mem)
    finally:
        eng.set_memory_budget(0)
        eng.set_host_budget(0)
