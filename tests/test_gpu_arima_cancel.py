"""Cancel and progress of ARIMA jobs (tad_cancel, tad_job_progress): the fit kernel stops at its next evaluation round once
a job is cancelled, so the job fails within one round of the cancel -- also inside one long series -- and the context goes
on with the next job; the fit counters add up over passes to the fits of the connections in the result."""
import threading
import time

import numpy as np
import pytest

from theia_b200 import synth
from tests.util import assert_same_rows

pytestmark = pytest.mark.gpu

TAD_ERR_CANCELLED = -6
MB = 1 << 20
BUDGET_2 = 150 * MB          # 2M-row host tables: two passes or more (as in test_gpu_passes.py)
KEY = ("src_ip", "dst_ip", "src_port", "dst_port", "proto", "flow_start")
# Sized on an H100 80GB HBM3 (400 W): the long table's fit phase takes 10.4 s.  The long connection's fits alone take far
# longer than the test waits: its longest fits come first, and one of them is tens of evaluation rounds over ~4,000 points.
LONG_SERIES = 150_000        # x 100 points
LONG_POINTS = 4_000          # one connection of this many points among 2,000 of 100


@pytest.fixture(scope="module")
def eng():
    """A context of its own: the jobs cancelled here and the budgets set here stay off the session's engine."""
    from theia_b200.engine import TadEngine
    e = TadEngine(device=0)
    yield e
    e.close()


def _device_table(parts):
    """DeviceColumns over the concatenation of make_flows_torch(series, points, seed, noisy=True) tables."""
    import torch
    from theia_b200.engine import DeviceColumns
    ts = [synth.make_flows_torch(s, p, seed=seed, device="cuda", noisy=True) for s, p, seed in parts]
    cols = {k: torch.cat([t[k] for t in ts]).contiguous() for k in ts[0]}
    torch.cuda.synchronize()
    d = DeviceColumns(int(cols["value"].numel()), {k: v.data_ptr() for k, v in cols.items()})
    d.keepalive = cols
    return d


def _host_table(series, points, seed):
    t = synth.make_flows_torch(series, points, seed=seed, device="cuda", noisy=True)
    return {k: t[k].cpu().numpy().view(dt) for k, dt in synth.COLUMN_DTYPES.items()}


def _result_connections(rows):
    """Points of every connection of an emit_all result (every point of a connection is a row)."""
    keys = np.stack([rows[k].astype(np.uint64) for k in KEY], axis=1)
    return np.unique(keys, axis=0, return_counts=True)[1]


def _check_fits(p, rows, st, points=100):
    """Every connection of these tables has `points` points and a Box-Cox lambda, so each is fitted (points - 3 fits); a
    connection whose forecasts do not transform back to finite values gives no rows but was fitted all the same."""
    n = _result_connections(rows)
    assert (n == points).all()
    assert p["fits_done"] == p["fits_total"] == st["series"] * (points - 3) >= len(n) * (points - 3) > 0


def _run(eng, cols, algo, **kw):
    job = eng.submit(cols, algo=algo, tad_id="cancel", **kw)
    try:
        st = job.wait()
        return job.result(), st, job.progress()
    finally:
        job.release()


def _wait_fitting(job, timeout=120.0):
    t0 = time.time()
    while job.progress()["fits_done"] == 0:
        assert job.poll()["state"] in ("SCHEDULED", "RUNNING"), job.poll()
        assert time.time() - t0 < timeout, "the fit phase did not start"
        time.sleep(0.005)


def test_progress_while_fitting(eng):
    cols = _device_table([(50_000, 100, 11)])
    job = eng.submit(cols, algo="ARIMA", tad_id="progress", emit_all=True)
    samples, stop = [], threading.Event()

    def sample():
        while not stop.is_set():
            samples.append(job.progress())
            time.sleep(0.02)
    th = threading.Thread(target=sample)
    th.start()
    try:
        st = job.wait()
    finally:
        stop.set()
        th.join()
    rows, end = job.result(), job.progress()
    job.release()
    print("progress: %d samples over a detect phase of %.0f ms" % (len(samples), st["phase_ms"]["detect"]))
    done = [s["fits_done"] for s in samples]
    assert done == sorted(done)
    assert all(s["fits_done"] <= s["fits_total"] for s in samples if s["fits_total"] > 0)
    assert any(0 < s["fits_done"] < s["fits_total"] for s in samples)
    _check_fits(end, rows, st)
    assert end["passes_done"] == end["passes"] == 1


def test_cancel_mid_fit_frees_the_context(eng):
    small = _device_table([(2_000, 100, 12)])
    ewma_cols = _device_table([(2_000, 100, 13)])
    before = [_run(eng, small, "ARIMA", emit_all=True)[0], _run(eng, ewma_cols, "EWMA")[0]]
    long_cols = _device_table([(LONG_SERIES, 100, 14)])
    job = eng.submit(long_cols, algo="ARIMA", tad_id="long")
    queued = eng.submit(ewma_cols, algo="EWMA", tad_id="queued")
    try:
        _wait_fitting(job)
        t0 = time.time()
        job.cancel()
        st = job.wait(check=False)
        dt = time.time() - t0
        p = job.progress()
        print("cancel -> FAILED in %.3f s at %d of %d fits" % (dt, p["fits_done"], p["fits_total"]))
        assert st["state"] == "FAILED" and st["error"] == TAD_ERR_CANCELLED, st
        assert dt < 1.0
        assert p["fits_done"] < p["fits_total"]
        assert queued.wait()["state"] == "COMPLETED"
    finally:
        job.release()
        queued.release()
    after = [_run(eng, small, "ARIMA", emit_all=True)[0], _run(eng, ewma_cols, "EWMA")[0]]
    for a, b, what in zip(before, after, ("ARIMA", "EWMA")):
        assert_same_rows(b, a, what=what + " after a cancelled job")


def test_cancel_within_one_long_series(eng):
    """One connection holds the fit phase for minutes: a per-series bound would wait for all of it, and even one of its
    ~4,000-point fits takes about a second; the cancel is seen at the next evaluation round."""
    cols = _device_table([(2_000, 100, 15), (1, LONG_POINTS, 16)])
    job = eng.submit(cols, algo="ARIMA", tad_id="long-series")
    try:
        _wait_fitting(job)
        time.sleep(1.0)                          # the short series are done by now; the long one is being fitted
        p0 = job.progress()
        t0 = time.time()
        job.cancel()
        st = job.wait(check=False)
        dt = time.time() - t0
        p = job.progress()
        print("long series: cancel -> FAILED in %.3f s at %d of %d fits (%d at the cancel)"
              % (dt, p["fits_done"], p["fits_total"], p0["fits_done"]))
        assert st["state"] == "FAILED" and st["error"] == TAD_ERR_CANCELLED, st
        assert p0["fits_done"] < p["fits_total"] - (LONG_POINTS - 3) // 2      # most of the long series was still to fit
        assert dt < 1.0
    finally:
        job.release()


def _run_budget(eng, table, budget, algo, **kw):
    seen = {}

    def on_job(j):
        if j is None:
            seen["progress"] = seen["job"].progress()
        else:
            seen["job"] = j
    rows, st = eng.run(table, on_job=on_job, memory_budget=budget, algo=algo, tad_id="passes", **kw)
    return rows, st, seen["progress"]


def test_progress_over_passes(eng):
    t = _host_table(20_000, 100, seed=17)
    ref, st_ref, p_ref = _run_budget(eng, t, 0, "ARIMA", emit_all=True)
    got, st, p = _run_budget(eng, t, BUDGET_2, "ARIMA", emit_all=True)
    eng.set_memory_budget(0)
    assert st_ref["memory"]["passes"] == 1 and st["memory"]["passes"] >= 2
    assert p_ref["passes_done"] == p_ref["passes"] == 1
    assert p["passes_done"] == p["passes"] == st["memory"]["passes"]
    _check_fits(p_ref, ref, st_ref)
    assert (p["fits_done"], p["fits_total"]) == (p_ref["fits_done"], p_ref["fits_total"])
    assert_same_rows(got, ref, what="ARIMA in %d passes vs one" % p["passes"])


@pytest.mark.parametrize("algo", ["EWMA", "DBSCAN"])
def test_other_algorithms_report_no_fits(eng, algo):
    t = synth.make_flows(20_000, 100, seed=18)
    _, st1, p1 = _run_budget(eng, t, 0, algo)
    _, st2, p2 = _run_budget(eng, t, BUDGET_2, algo)
    eng.set_memory_budget(0)
    assert (p1["fits_done"], p1["fits_total"], p2["fits_done"], p2["fits_total"]) == (0, 0, 0, 0)
    assert p1["passes_done"] == p1["passes"] == st1["memory"]["passes"] == 1
    assert p2["passes_done"] == p2["passes"] == st2["memory"]["passes"] >= 2


def _flows(series, points, seed):
    t = _host_table(series, points, seed)
    return {"sourceIP": t["src_ip"], "destinationIP": t["dst_ip"], "sourceTransportPort": t["src_port"],
            "destinationTransportPort": t["dst_port"], "protocolIdentifier": t["proto"], "flowStartSeconds": t["flow_start"],
            "flowEndSeconds": t["flow_end"], "throughput": t["value"]}


def test_controller_delete_of_a_fitting_job(eng):
    from theia_b200 import controller as ctl
    c = ctl.AnomalyDetectorController(eng)
    long_name = "tad-5ca1ab1e-0000-4000-8000-0000000000c1"
    next_name = "tad-5ca1ab1e-0000-4000-8000-0000000000c2"
    c.create(long_name, ctl.TADSpec(jobType="ARIMA"))
    c.create(next_name, ctl.TADSpec(jobType="EWMA"))
    assert c.sync(long_name, flows=_flows(50_000, 100, 19)).state == "SCHEDULED"
    run = c._jobs[long_name]
    t0 = time.time()
    while True:
        with run.lock:
            p = run.handle.progress() if run.handle is not None else None
        if p is not None and p["fits_done"] > 0:
            break
        assert not run.done.is_set() and time.time() - t0 < 300, "the fit phase did not start"
        time.sleep(0.005)
    assert c.sync(next_name, flows=_flows(2_000, 100, 20)).state == "SCHEDULED"
    t0 = time.time()
    c.delete(long_name)
    dt = time.time() - t0
    print("controller delete of a fitting ARIMA job: %.3f s" % dt)
    assert dt < 1.0 and long_name not in c.crs
    assert c.wait(next_name).state == "COMPLETED"
    c.delete(next_name)
