"""The job entry point on streamed input with the real engine: main() over a 2M-row ClickHouse double in 65,536-row blocks,
TAD_STREAM_INPUT=1 against the default one-shot path, with no budget, with a device budget that forces hash-range passes
(one SELECT per pass) and with the same budget plus a host row store (one SELECT)."""
import numpy as np
import pytest

from theia_b200 import anomaly_detection as ad
from theia_b200 import clickhouse_native as chn

from .test_gpu_stream import BUDGET_4
from .test_job_entry_stream import TableTransport, make_table

pytestmark = pytest.mark.gpu

HOST = 256 << 20                      # holds the 2M filtered rows (32 B each)
BLOCK = 65536


@pytest.fixture(scope="module")
def eng():
    """A context of its own: the budgets set here must not reach the session's engine."""
    from theia_b200.engine import TadEngine
    e = TadEngine(device=0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def table():
    return make_table(series=20000, points=100, seed=84)          # 2M rows


def canonical_rows(body):
    """The INSERT body's columns as text, rows in sorted order (row order is not part of the result)."""
    got = chn.read_native(body)
    text = {c: np.asarray(got[c]).astype(str) for c in sorted(got)}
    order = np.lexsort(tuple(text.values()))
    return {c: v[order] for c, v in text.items()}


def same(a, b):
    return a.keys() == b.keys() and all(np.array_equal(a[c], b[c]) for c in a)


class _Recording:
    """The engine, with the memory report of every streamed job kept (main() only returns an exit code)."""

    def __init__(self, eng):
        self.eng, self.memory = eng, []

    def __getattr__(self, name):
        return getattr(self.eng, name)

    def submit_stream(self, **kw):
        job = self.eng.submit_stream(**kw)
        wait = job.wait

        def wait_and_report(*a, **k):
            st = wait(*a, **k)
            self.memory.append(job.memory())
            return st
        job.wait = wait_and_report
        return job


@pytest.mark.parametrize("algo", ["EWMA", "DBSCAN"])
def test_streamed_entry_equals_the_one_shot_entry(eng, table, algo, monkeypatch):
    argv = ["--algo", algo, "--id", "gpu-stream", "--ns-ignore-list", '["kube-system"]']
    monkeypatch.delenv("TAD_STREAM_INPUT", raising=False)
    monkeypatch.delenv("TAD_HOST_BUDGET", raising=False)
    eng.set_memory_budget(0)
    eng.set_host_budget(0)
    tr = TableTransport(table, block_rows=BLOCK)
    assert ad.main(argv, engine=eng, transport=tr) == 0
    want = canonical_rows(tr.inserts[0][1])
    assert len(want["id"]) > 1
    monkeypatch.setenv("TAD_STREAM_INPUT", "1")
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
            what = (algo, budget, host)
            assert same(canonical_rows(tr.inserts[0][1]), want), what
            (mem,) = rec.memory
            assert tr.counts and len(tr.selects) == (1 if host or not budget else mem["passes"]), (what, mem)
            if budget:
                assert mem["passes"] >= 4 and mem["peak_workspace_bytes"] <= budget, (what, mem)
            if host:
                assert mem["stored_rows"] > 0 and len(tr.selects) == 1, (what, mem)
            else:
                assert mem["stored_rows"] == 0, (what, mem)
    finally:
        eng.set_memory_budget(0)
        eng.set_host_budget(0)


def test_pushdown_streamed_entry_equals_the_one_shot_entry(eng, table, monkeypatch):
    monkeypatch.setenv("TAD_IPV4_PUSHDOWN", "1")
    argv = ["--algo", "EWMA", "--id", "gpu-pushdown"]
    out = []
    for stream in ("0", "1"):
        monkeypatch.setenv("TAD_STREAM_INPUT", stream)
        tr = TableTransport(table, block_rows=BLOCK)
        assert ad.main(argv, engine=eng, transport=tr) == 0
        assert all("IPv4StringToNum" in q for q in tr.selects)
        out.append(canonical_rows(tr.inserts[0][1]))
    assert same(out[0], out[1]) and len(out[0]["id"]) > 1
    assert np.asarray(table["sourceIP"]).dtype == np.uint32
