"""Host row store (tad_set_host_budget): a streamed job that needs several hash-range passes keeps its first round's rows
in pinned host pages and loads every pass from them, so the caller delivers its rows once.  Every result equals a
one-shot run of the whole table bit for bit, on all 11 result columns and on the status counters."""
import ctypes as C

import numpy as np
import pytest

from theia_b200 import synth
from tests.test_gpu_stream import BUDGET_2, BUDGET_4, block_source, device_cols
from tests.util import assert_same_rows, oracle_rows

pytestmark = pytest.mark.gpu

MB = 1 << 20
HOST = 1 << 30                     # holds the filtered rows of every table here (32 B per row)
COUNTS = ("rows_in", "rows_kept", "points", "series", "result_rows")
ERR_INVALID_ARG, ERR_STATE, ERR_CANCELLED = -1, -5, -6


@pytest.fixture(scope="module")
def eng():
    """A context of its own: the budgets set here must not reach the session's engine."""
    from theia_b200.engine import TadEngine
    e = TadEngine(device=0)
    yield e
    e.close()


def one_shot(eng, table, **kw):
    eng.set_memory_budget(0)
    eng.set_host_budget(0)
    return eng.run(table, tad_id="one-shot", **kw)


def streamed(eng, table, sizes, kind, budget, host=HOST, **kw):
    eng.set_memory_budget(budget)
    eng.set_host_budget(host)
    factory = block_source(eng, table, sizes, kind)
    try:
        return eng.run_stream(factory, tad_id="stored", **kw)
    finally:
        factory.free()
        eng.set_host_budget(0)


def same(got, st, ref, st_ref, what):
    for k in COUNTS:
        assert st[k] == st_ref[k], (what, k, st[k], st_ref[k])
    assert_same_rows(got, ref, what=what)


def one_round(st, budget, host, min_passes):
    mem = st["memory"]
    assert st["state"] == "COMPLETED" and st["rounds"] == 1, (st["rounds"], mem)
    assert mem["passes"] >= min_passes, mem
    assert mem["stored_rows"] == st["rows_kept"] > 0, (mem, st["rows_kept"])
    assert 0 < mem["peak_host_bytes"] <= host, mem
    assert mem["peak_workspace_bytes"] <= budget, mem


BIG = synth.make_flows(20000, 100, seed=84)           # 2M rows
_REF = {}


def big_ref(eng):
    if "big" not in _REF:
        _REF["big"] = one_shot(eng, BIG)
    return _REF["big"]


@pytest.mark.parametrize("sizes,kind,budget,min_passes", [
    (65536, "pinned", BUDGET_2, 2), (65536, "pinned", BUDGET_4, 4), (65536, "pageable", BUDGET_2, 2),
    ("uneven", "pageable", BUDGET_4, 4), (65536, "device", BUDGET_2, 2), ("uneven", "device", BUDGET_4, 4),
    ("uneven", "pinned", BUDGET_4, 4)])
def test_one_round_under_a_budget(eng, sizes, kind, budget, min_passes):
    ref, st_ref = big_ref(eng)
    n = len(BIG["flow_end"])
    got, st = streamed(eng, BIG, sizes, kind, budget, rows_hint=n)
    one_round(st, budget, HOST, min_passes)
    same(got, st, ref, st_ref, "store %s %s %d" % (sizes, kind, budget))


@pytest.mark.parametrize("kind", ["pinned", "device"])
@pytest.mark.parametrize("hint_div", [0, 10])
def test_pass_columns_overflow_switches_to_the_store(eng, kind, hint_div):
    """No hint, or one 10x too low: the first round fills the pass columns, overflows them, moves their rows to the store
    and goes on there.  Still one round."""
    ref, st_ref = big_ref(eng)
    n = len(BIG["flow_end"])
    got, st = streamed(eng, BIG, 65536, kind, BUDGET_4, rows_hint=n // hint_div if hint_div else 0)
    one_round(st, BUDGET_4, HOST, 4)
    same(got, st, ref, st_ref, "switch %s hint/%d" % (kind, hint_div))


def test_overestimated_hint_costs_nothing(eng):
    ref, st_ref = big_ref(eng)
    n = len(BIG["flow_end"])
    _, st_exact = streamed(eng, BIG, 65536, "pinned", BUDGET_4, rows_hint=n)
    got, st = streamed(eng, BIG, 65536, "pinned", BUDGET_4, rows_hint=8 * n)
    one_round(st, BUDGET_4, HOST, 4)
    assert st["memory"]["passes"] == st_exact["memory"]["passes"], (st["memory"], st_exact["memory"])
    same(got, st, ref, st_ref, "hint x8")


def test_dbscan(eng):
    ref, st_ref = one_shot(eng, BIG, algo="DBSCAN")
    got, st = streamed(eng, BIG, 65536, "pinned", BUDGET_2, algo="DBSCAN", rows_hint=len(BIG["flow_end"]))
    one_round(st, BUDGET_2, HOST, 2)
    same(got, st, ref, st_ref, "DBSCAN")


def test_arima(eng):
    t = synth.make_flows(10000, 100, seed=93, dup_frac=0.1)
    ref, st_ref = one_shot(eng, t, algo="ARIMA")
    got, st = streamed(eng, t, 65536, "pageable", BUDGET_4, algo="ARIMA", rows_hint=len(t["flow_end"]))
    one_round(st, BUDGET_4, HOST, 2)
    same(got, st, ref, st_ref, "ARIMA")


@pytest.mark.parametrize("kind", ["pageable", "pinned"])
def test_filters_and_sum_reducer(eng, kind):
    t = dict(BIG)
    rng = np.random.default_rng(94)
    n = len(t["value"])
    t["src_ns"] = rng.integers(0, 6, n).astype(np.uint32)
    t["dst_ns"] = rng.integers(0, 6, n).astype(np.uint32)
    kw = dict(reducer=1, start_time=synth.T0 + 600, end_time=synth.T0 + 3000, ns_ignore=(1, 4), emit_all=True)
    ref, st_ref = one_shot(eng, t, **kw)
    got, st = streamed(eng, t, "uneven", kind, BUDGET_4, rows_hint=n, **kw)
    assert st["rows_kept"] < st["rows_in"] == n
    one_round(st, BUDGET_4, HOST, 2)
    same(got, st, ref, st_ref, "filters %s" % kind)


def test_spill_and_pass_split_from_the_store(eng):
    """Connections of 6000 points only: every row takes the spill path, and under BUDGET_4 a pass's spill scratch does not
    fit, so passes split into (v, 2M) and (v + M, 2M).  Without a store every split costs two rounds more, which gives the
    planned P and the splits; with the store the halves are loaded from it in the one round."""
    t = synth.make_flows(400, 6000, seed=86)
    n = len(t["flow_end"])
    ref, st_ref = one_shot(eng, t, emit_all=True)
    got0, st0 = streamed(eng, t, 65536, "pinned", BUDGET_4, host=0, rows_hint=n, emit_all=True)
    splits = st0["rounds"] - st0["memory"]["passes"]
    planned = st0["memory"]["passes"] - splits
    assert splits > 0 and planned >= 2, (st0["rounds"], st0["memory"])
    same(got0, st0, ref, st_ref, "spill and split, no store")
    got, st = streamed(eng, t, 65536, "pinned", BUDGET_4, rows_hint=n, emit_all=True)
    assert st["spill_rows"] > 0
    one_round(st, BUDGET_4, HOST, 2)
    assert st["memory"]["passes"] > planned, (st["memory"], planned)     # at least one pass split, served from the store
    same(got, st, ref, st_ref, "spill and split from the store")


def test_source_that_changes_between_reads(eng):
    """With the store the source is read once: a second read would deliver other rows, and is never asked for."""
    first = synth.make_flows(20000, 100, seed=95)
    second = synth.make_flows(20000, 100, seed=96)
    calls = [0]

    def factory():
        t = first if calls[0] == 0 else second
        calls[0] += 1
        n = len(t["flow_end"])
        for lo in range(0, n, 65536):
            yield {k: v[lo:lo + 65536] for k, v in t.items()}

    ref, st_ref = one_shot(eng, first)
    eng.set_memory_budget(BUDGET_4)
    eng.set_host_budget(HOST)
    try:
        got, st = eng.run_stream(factory, tad_id="changing", rows_hint=len(first["flow_end"]))
    finally:
        eng.set_host_budget(0)
    assert calls[0] == 1
    one_round(st, BUDGET_4, HOST, 4)
    same(got, st, ref, st_ref, "changing source")


def test_store_too_small_falls_back(eng):
    """64 MiB of store cannot hold 3M rows: the job drops the store and runs as without one."""
    t = synth.make_flows(30000, 100, seed=92, dup_frac=0.1)
    ref, st_ref = one_shot(eng, t, emit_all=True)
    got0, st0 = streamed(eng, t, 65536, "pinned", BUDGET_4, host=0, rows_hint=0, emit_all=True)
    got, st = streamed(eng, t, 65536, "pinned", BUDGET_4, host=64 * MB, rows_hint=0, emit_all=True)
    assert st0["rounds"] > 1
    assert st["rounds"] == st0["rounds"], (st["rounds"], st0["rounds"])
    assert st["memory"]["passes"] == st0["memory"]["passes"]
    # the store was tried (the budget was 0 before this job, so every pinned byte is this job's) and dropped
    assert st["memory"]["stored_rows"] == 0 and 0 < st["memory"]["peak_host_bytes"] <= 64 * MB, st["memory"]
    same(got, st, ref, st_ref, "fallback")
    same(got0, st0, ref, st_ref, "no store")


TABLE = synth.make_flows(300, 40, seed=81, dup_frac=0.25)


def test_one_pass_job_does_not_touch_the_store(eng):
    n = len(TABLE["flow_end"])
    got0, st0 = streamed(eng, TABLE, 65536, "pinned", 0, host=0, rows_hint=n, emit_all=True)
    got, st = streamed(eng, TABLE, 65536, "pinned", 0, host=HOST, rows_hint=n, emit_all=True)
    assert st["rounds"] == 1 and st["memory"]["passes"] == 1
    assert st["memory"]["stored_rows"] == 0
    assert st["gpu_launches"] == st0["gpu_launches"], (st["gpu_launches"], st0["gpu_launches"])
    same(got, st, got0, st0, "P = 1")
    want, _, _ = oracle_rows(TABLE, "EWMA", emit_all=True)
    assert_same_rows(got, want, what="P = 1 vs oracle")


def test_submit_jobs_do_not_use_the_store(eng):
    ref, st_ref = big_ref(eng)
    eng.set_host_budget(HOST)
    try:
        got, st = eng.run(BIG, memory_budget=BUDGET_4, tad_id="host input")
        assert st["memory"]["passes"] >= 4 and st["memory"]["stored_rows"] == 0, st["memory"]
        same(got, st, ref, st_ref, "tad_submit host input")
        d = device_cols(BIG)
        job = eng.submit(d, tad_id="device input")
        try:
            st = job.wait()
            mem = job.memory()
            assert mem["passes"] >= 4 and mem["stored_rows"] == 0, mem
            same(job.result(), st, ref, st_ref, "tad_submit device input")
        finally:
            job.release()
    finally:
        eng.set_host_budget(0)
        eng.set_memory_budget(0)


def test_cancel_while_filling_the_store():
    from theia_b200.engine import TadEngine, TadError
    e = TadEngine(device=0, memory_budget=BUDGET_4, host_budget=HOST)
    try:
        n = len(BIG["flow_end"])
        job = e.submit_stream(rows_hint=n, tad_id="cancel")
        for lo in range(0, 8 * 65536, 65536):
            job.push({k: v[lo:lo + 65536] for k, v in BIG.items()})
        job.cancel()
        with pytest.raises(TadError) as exc:
            job.push({k: v[8 * 65536:9 * 65536] for k, v in BIG.items()})
        assert exc.value.code == ERR_CANCELLED
        assert job.wait(check=False)["state"] == "FAILED"
        job.release()
        ref, st_ref = big_ref(e)
        e.set_memory_budget(BUDGET_4)
        e.set_host_budget(HOST)
        factory = block_source(e, BIG, 65536, "pinned")
        try:
            got, st = e.run_stream(factory, tad_id="after cancel", rows_hint=n)
        finally:
            factory.free()
        one_round(st, BUDGET_4, HOST, 4)
        same(got, st, ref, st_ref, "after cancel")
        e.set_host_budget(0)
    finally:
        e.close()


def _feed_rounds(job, table):
    rounds, again = 0, True
    while again:
        for lo in range(0, len(table["flow_end"]), 65536):
            job.push({k: v[lo:lo + 65536] for k, v in table.items()})
        again = job.end()
        rounds += 1
    return rounds


@pytest.mark.parametrize("before,after", [(0, HOST), (HOST, 0)])
def test_budget_changed_after_the_job_started(eng, before, after):
    """A job reads the host budget once, when the worker starts it: a streamed job on an idle context starts at submit,
    before its first block, and a budget set after that applies to the next job only."""
    import time
    ref, st_ref = big_ref(eng)
    n = len(BIG["flow_end"])
    eng.set_memory_budget(BUDGET_4)
    eng.set_host_budget(before)
    job = eng.submit_stream(rows_hint=n, tad_id="budget after start")
    try:
        time.sleep(0.3)                     # the worker has taken the job and waits for its first block
        eng.set_host_budget(after)
        rounds = _feed_rounds(job, BIG)
        st = job.wait()
        mem = job.memory()
        same(job.result(), st, ref, st_ref, "budget %d -> %d" % (before, after))
    finally:
        job.release()
        eng.set_host_budget(0)
    if before:
        assert rounds == 1 and mem["stored_rows"] == st["rows_kept"] and mem["peak_host_bytes"] <= before, mem
    else:
        assert rounds == mem["passes"] >= 4 and mem["stored_rows"] == 0 and mem["peak_host_bytes"] == 0, (rounds, mem)


def test_errors(eng):
    from theia_b200.engine import TadError
    with pytest.raises(TadError) as exc:
        eng.set_host_budget(32 * MB)
    assert exc.value.code == ERR_INVALID_ARG
    eng.set_host_budget(0)
    job = eng.submit_stream(tad_id="not completed")
    try:
        job.push({k: v[:1000] for k, v in TABLE.items()})
        stored, peak = C.c_uint64(), C.c_uint64()
        assert eng.lib.tad_job_host_memory(job.h, C.byref(stored), C.byref(peak)) == ERR_STATE
        assert job.end() is False
        job.wait()
        assert job.memory()["stored_rows"] == 0
    finally:
        job.release()
