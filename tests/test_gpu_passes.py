"""Single-GPU jobs in hash-range passes under a memory budget (tad_set_memory_budget): the rows and counts of every pass
split equal the one-pass run and the C oracle, the workspace stays inside the budget, and a job larger than device
memory runs without one."""
import os

import numpy as np
import pytest

from theia_b200 import synth
from tests.util import assert_same_rows, oracle_rows

pytestmark = pytest.mark.gpu

MB = 1 << 20
BUDGET_2 = 150 * MB          # 2M-row host tables: two passes or more
BUDGET_4 = 64 * MB           # the floor: four passes or more
DEVICE_BUDGET_2 = 100 * MB   # device-resident input needs no staged copy of the columns
COUNTS = ("rows_in", "rows_kept", "rows_owned", "points", "series", "result_rows")
_SIGNED = {np.dtype(np.uint32): np.int32, np.dtype(np.uint16): np.int16, np.dtype(np.uint64): np.int64,
           np.dtype(np.uint8): np.uint8}


@pytest.fixture(scope="module")
def eng():
    """A context of its own: the budgets set here must not reach the session's engine."""
    from theia_b200.engine import TadEngine
    e = TadEngine(device=0)
    yield e
    e.close()


def _device_cols(table):
    import torch
    from theia_b200.engine import DeviceColumns
    ts = {k: torch.from_numpy(np.ascontiguousarray(v).view(_SIGNED[v.dtype])).cuda() for k, v in table.items()
          if v is not None and k not in ("src_ns", "dst_ns")}
    d = DeviceColumns(len(table["flow_end"]), {k: t.data_ptr() for k, t in ts.items()})
    d.keepalive = ts
    return d


def run(eng, table, budget=0, device=False, algo="EWMA", check=True, **kw):
    eng.set_memory_budget(budget)
    cols = _device_cols(table) if device else eng.columns_from_numpy(table)
    job = eng.submit(cols, algo=algo, tad_id="passes", **kw)
    try:
        st = job.wait(check=check)
        if st["state"] != "COMPLETED":
            return None, st, None
        return job.result(), st, job.memory()
    finally:
        job.release()
        cols.free()


def check_against_one_pass(eng, table, budgets, device=False, algo="EWMA", oracle=True, **kw):
    ref, st_ref, mem_ref = run(eng, table, 0, device, algo, **kw)
    assert mem_ref["passes"] == 1
    if oracle:
        okw = {k: v for k, v in kw.items() if k in ("emit_all", "reducer", "start_time", "end_time")}
        want, ns, npts = oracle_rows(table, algo, **okw)
        assert st_ref["series"] == ns and st_ref["points"] == npts
    for budget, min_passes in budgets:
        got, st, mem = run(eng, table, budget, device, algo, **kw)
        what = "%s budget %d device=%s %s" % (algo, budget, device, kw)
        assert mem["passes"] >= min_passes, (what, mem)
        assert mem["peak_workspace_bytes"] <= budget, (what, mem)
        assert st["completed_stages"] == 6
        for k in COUNTS:
            assert st[k] == st_ref[k], (what, k, st[k], st_ref[k])
        assert_same_rows(got, ref, what=what + " vs one pass")          # bit for bit, canonical order
        if oracle:
            assert_same_rows(got, want, what=what + " vs oracle")
    return ref, st_ref


@pytest.mark.parametrize("algo", ["EWMA", "DBSCAN"])
@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("emit_all", [False, True])
def test_parity_across_passes(eng, algo, device, emit_all):
    t = synth.make_flows(20000, 100, seed=61)                      # 2M rows
    check_against_one_pass(eng, t, [(DEVICE_BUDGET_2 if device else BUDGET_2, 2), (BUDGET_4, 4)], device=device, algo=algo,
                           emit_all=emit_all)


def test_parity_across_passes_10m_rows(eng):
    t = synth.make_flows(100000, 100, seed=62, ragged=True)        # ~10M rows
    check_against_one_pass(eng, t, [(400 * MB, 2), (200 * MB, 4)], device=True)


def test_arima_bit_identical_across_passes(eng):
    """A series' fits do not depend on which other series share the launch: ARIMA in passes equals its one-pass run bit
    for bit (the one-pass run's agreement with the oracle is covered by test_gpu_parity)."""
    import torch
    t = synth.torch_cols_to_numpy(synth.make_flows_torch(20000, 40, seed=63, device=torch.device("cuda", 0), noisy=True))
    check_against_one_pass(eng, t, [(BUDGET_4, 2)], algo="ARIMA", oracle=False, emit_all=True)


def test_filters_and_reducer_under_passes(eng):
    t = synth.make_flows(20000, 100, seed=64, dup_frac=0.3)
    check_against_one_pass(eng, t, [(BUDGET_4, 4)], start_time=synth.T0 + 600, end_time=synth.T0 + 3600, emit_all=True)
    check_against_one_pass(eng, t, [(BUDGET_4, 4)], reducer=1, emit_all=True)
    # ns_ignore: the split kernel applies it; the namespace columns never reach the pass columns
    rng = np.random.default_rng(64)
    n = len(t["value"])
    t["src_ns"] = rng.integers(0, 6, n).astype(np.uint32)
    t["dst_ns"] = rng.integers(0, 6, n).astype(np.uint32)
    ignore = (1, 4)
    ref, st_ref, _ = run(eng, t, 0, ns_ignore=ignore, emit_all=True)
    got, st, mem = run(eng, t, BUDGET_4, ns_ignore=ignore, emit_all=True)
    assert mem["passes"] >= 4 and mem["peak_workspace_bytes"] <= BUDGET_4
    keep = ~np.isin(t["src_ns"], ignore) & ~np.isin(t["dst_ns"], ignore)
    assert st["rows_kept"] == st_ref["rows_kept"] == int(keep.sum())
    assert_same_rows(got, ref, what="ns_ignore vs one pass")
    want, _, _ = oracle_rows({k: v[keep] for k, v in t.items() if k not in ("src_ns", "dst_ns")}, "EWMA", emit_all=True)
    assert_same_rows(got, want, what="ns_ignore vs oracle")


def test_spill_under_passes(eng):
    """Connections of more than 4096 points take the oversized-bucket path inside their pass."""
    small = synth.make_flows(20000, 100, seed=65)
    big = synth.make_flows(30, 6000, seed=66)
    t = {k: np.concatenate([small[k], big[k]]) for k in small}
    _, st = check_against_one_pass(eng, t, [(BUDGET_4, 4)], emit_all=True)
    assert st["spill_rows"] > 0


def test_lowered_budget_frees_the_workspace():
    import torch
    from theia_b200.engine import TadEngine
    t = synth.make_flows(20000, 100, seed=67)
    with TadEngine(device=0) as e:
        cols_t = synth.make_flows_torch(300000, 100, seed=67, device=torch.device("cuda", 0))
        from theia_b200.engine import DeviceColumns
        d = DeviceColumns(30_000_000, {k: v.data_ptr() for k, v in cols_t.items()})
        job = e.submit(d, algo="EWMA")
        job.wait()
        big_peak = job.memory()["peak_workspace_bytes"]
        job.release()
        del cols_t, d
        torch.cuda.empty_cache()
        assert big_peak > 4 * BUDGET_4
        got, st, mem = run(e, t, BUDGET_4)
        assert mem["peak_workspace_bytes"] <= BUDGET_4 and mem["passes"] >= 4
        ref, _, _ = run(e, t, 0)
        assert_same_rows(got, ref, what="after lowering the budget")


def test_impossible_budget_fails_then_context_recovers(eng):
    from theia_b200.engine import TadError
    one = synth.make_flows(1, 2_000_000, seed=68)             # one connection, ~2M points: no split can shrink it
    _, st, _ = run(eng, one, BUDGET_4, check=False)
    assert st["state"] == "FAILED" and st["error"] == -3, st           # TAD_ERR_NOMEM
    assert "bytes" in st["err_msg"] and "budget" in st["err_msg"], st["err_msg"]
    t = synth.make_flows(300, 20, seed=69)
    got, st, mem = run(eng, t, BUDGET_4, emit_all=True)
    want, _, _ = oracle_rows(t, "EWMA", emit_all=True)
    assert_same_rows(got, want, what="after a failed job")
    with pytest.raises(TadError):
        eng.set_memory_budget(BUDGET_4 - 1)                          # below the floor


def test_default_budget_runs_today_s_jobs_in_one_pass(eng):
    import torch
    eng.set_memory_budget(0)
    ref = __import__("json").load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_test_vectors.json")))
    for t in (synth.golden_e2e_table(ref["throughput_list"], duplicates=1), synth.make_flows(100, 100, seed=0)):
        _, st, mem = run(eng, t)
        assert mem["passes"] == 1
    free, _ = torch.cuda.mem_get_info()
    if free < 40e9:
        pytest.skip("configs[1] size needs ~40 GB of free HBM")
    from theia_b200.engine import DeviceColumns
    cols_t = synth.make_flows_torch(1_000_000, 100, seed=7, device=torch.device("cuda", 0))
    torch.cuda.synchronize()
    d = DeviceColumns(100_000_000, {k: v.data_ptr() for k, v in cols_t.items()})
    job = eng.submit(d, algo="EWMA")
    st = job.wait()
    assert job.memory()["passes"] == 1 and st["points"] == 100_000_000
    job.release()
    del cols_t
    torch.cuda.empty_cache()
