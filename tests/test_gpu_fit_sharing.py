"""Fit sharing (tad_set_fit_sharing): a long ARIMA fit yields to queued EWMA and DBSCAN jobs, which run in the reserve
while its buffers are parked, and resumes; every job's rows, and the ARIMA job's fit counts, equal those of a solo run."""
import time

import numpy as np
import pytest

from theia_b200 import synth
from tests.util import assert_same_rows

pytestmark = pytest.mark.gpu

TAD_ERR_INVALID_ARG = -1
TAD_ERR_CANCELLED = -6
MB = 1 << 20
RESERVE = 256 * MB
# the long table of tests/test_gpu_arima_cancel.py: its fit phase takes about 10 s on an H100
LONG_SERIES = 150_000
LONG_POINTS = 4_000
# one evaluation round of the 4,000-point connection: the cancel of tests/test_gpu_arima_cancel.py waits 21-23 ms for it
ROUND_S = 0.023
POLL_S = 0.005               # the worker's and the caller's 1 ms polls, and the park


@pytest.fixture(scope="module")
def eng():
    from theia_b200.engine import TadEngine
    e = TadEngine(device=0)
    yield e
    e.close()


def _device_table(parts):
    import torch
    from theia_b200.engine import DeviceColumns
    ts = [synth.make_flows_torch(s, p, seed=seed, device="cuda", noisy=True) for s, p, seed in parts]
    cols = {k: torch.cat([t[k] for t in ts]).contiguous() for k in ts[0]}
    torch.cuda.synchronize()
    d = DeviceColumns(int(cols["value"].numel()), {k: v.data_ptr() for k, v in cols.items()})
    d.keepalive = cols
    return d


def _host_table(parts):
    ts = [synth.make_flows_torch(s, p, seed=seed, device="cuda", noisy=True) for s, p, seed in parts]
    return {k: np.concatenate([t[k].cpu().numpy() for t in ts]).view(dt) for k, dt in synth.COLUMN_DTYPES.items()}


def _solo(eng, cols, algo, **kw):
    job = eng.submit(cols, algo=algo, tad_id="solo", **kw)
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
        time.sleep(0.002)


@pytest.fixture(scope="module")
def long_arima(eng):
    """The long table and its solo ARIMA run (sharing off)."""
    cols = _device_table([(LONG_SERIES, 100, 14)])
    rows, st, p = _solo(eng, cols, "ARIMA", emit_all=True)
    return cols, rows, st, p


def test_reserve_floor(eng):
    from theia_b200.engine import TadError
    for bad in (1, 64 * MB - 1):
        with pytest.raises(TadError) as e:
            eng.set_fit_sharing(bad)
        assert e.value.code == TAD_ERR_INVALID_ARG
    eng.set_fit_sharing(64 * MB)
    eng.set_fit_sharing(0)


def _check_arima(job, ref):
    _, rows_ref, st_ref, p_ref = ref
    st = job.wait()
    rows, p = job.result(), job.progress()
    assert_same_rows(rows, rows_ref, what="ARIMA beside other jobs")
    assert (p["fits_done"], p["fits_total"]) == (p_ref["fits_done"], p_ref["fits_total"])
    return st, job.yields()


def test_ewma_completes_while_the_fit_runs(eng, long_arima):
    ewma_cols = _device_table([(2_000, 100, 13)])
    ref_e = _solo(eng, ewma_cols, "EWMA")[0]
    eng.set_fit_sharing(RESERVE)
    job = eng.submit(long_arima[0], algo="ARIMA", tad_id="long", emit_all=True)
    try:
        _wait_fitting(job)
        time.sleep(0.5)
        t0 = time.time()
        q = eng.submit(ewma_cols, algo="EWMA", tad_id="beside")
        q.wait()
        dt = time.time() - t0
        state = job.poll()["state"]
        rows_q = q.result()
        q.release()
        st, y = _check_arima(job, long_arima)
    finally:
        eng.set_fit_sharing(0)
        job.release()
    print("EWMA beside the fit: %.3f s; ARIMA yields %d, parked %.1f ms, detect %.0f ms (solo %.0f ms)"
          % (dt, y["yields"], y["parked_ms"], st["phase_ms"]["detect"], long_arima[2]["phase_ms"]["detect"]))
    assert state == "RUNNING"
    assert dt < 1.0
    assert y["yields"] >= 1
    assert_same_rows(rows_q, ref_e, what="EWMA beside the fit")


def test_jobs_spread_over_the_fit_phase(eng, long_arima):
    tables = [(_device_table([(2_000, 100, 20 + k)]), "EWMA" if k % 2 == 0 else "DBSCAN") for k in range(5)]
    refs = [_solo(eng, c, a)[0] for c, a in tables]
    solo_detect_s = long_arima[2]["phase_ms"]["detect"] * 1e-3
    eng.set_fit_sharing(RESERVE)
    job = eng.submit(long_arima[0], algo="ARIMA", tad_id="long", emit_all=True)
    got = []
    try:
        _wait_fitting(job)
        t_fit = time.time()
        for k, (c, a) in enumerate(tables):
            time.sleep(solo_detect_s / 7)
            q = eng.submit(c, algo=a, tad_id="spread")
            q.wait()
            got.append(q.result())
            q.release()
        job.wait()
        wall = time.time() - t_fit          # before the comparison of its 1.5e7 rows
        st, y = _check_arima(job, long_arima)
    finally:
        eng.set_fit_sharing(0)
        job.release()
    print("5 jobs over the fit phase: ARIMA wall %.2f s from its first fit (solo detect %.2f s), %d yields, parked %.1f ms"
          % (wall, solo_detect_s, y["yields"], y["parked_ms"]))
    for g, r, (_, a) in zip(got, refs, tables):
        assert_same_rows(g, r, what=a + " spread over the fit phase")
    assert y["yields"] >= 1
    assert wall <= 2.0 * solo_detect_s + 1.0


def test_wait_behind_one_long_series(eng):
    """Only the 4,000-point connection is being fitted: the queued job waits for about one evaluation round of it."""
    from theia_b200.engine import TadEngine
    ewma_cols = _device_table([(2_000, 100, 13)])
    with TadEngine(device=0) as fresh:          # its run time on an empty workspace, as it runs beside the fit
        own_s = _solo(fresh, ewma_cols, "EWMA")[1]["total_ms"] * 1e-3
    cols = _device_table([(2_000, 100, 15), (1, LONG_POINTS, 16)])
    eng.set_fit_sharing(RESERVE)
    job = eng.submit(cols, algo="ARIMA", tad_id="long-series")
    try:
        _wait_fitting(job)
        time.sleep(1.0)                          # the short series are done: only the long one is being fitted
        t0 = time.time()
        q = eng.submit(ewma_cols, algo="EWMA", tad_id="behind-one-series")
        q.wait()
        dt = time.time() - t0
        q.release()
        assert job.poll()["state"] == "RUNNING"
        t0 = time.time()
        job.cancel()
        assert job.wait(check=False)["error"] == TAD_ERR_CANCELLED
        dc = time.time() - t0
    finally:
        eng.set_fit_sharing(0)
        job.release()
    print("EWMA behind one long series: %.1f ms (its own run %.1f ms); a cancel there: %.1f ms" % (dt * 1e3, own_s * 1e3, dc * 1e3))
    assert dt <= ROUND_S + own_s + POLL_S


def test_cancel_while_parked(eng, long_arima):
    small = _device_table([(2_000, 100, 12)])
    before = _solo(eng, small, "ARIMA", emit_all=True)[0]
    # a job that runs long enough to be seen running: a host table in several passes of the reserve
    big = _host_table([(100_000, 100, 30)])
    cols = eng.columns_from_numpy(big)
    eng.set_memory_budget(0)
    ref_q = _solo(eng, cols, "EWMA")[0]
    eng.set_fit_sharing(64 * MB)
    t_job = time.time()
    job = eng.submit(long_arima[0], algo="ARIMA", tad_id="long")
    try:
        _wait_fitting(job)
        t_q = time.time()
        q = eng.submit(cols, algo="EWMA", tad_id="in-its-place")
        t0 = time.time()
        while q.poll()["state"] != "RUNNING":
            assert time.time() - t0 < 5.0, q.poll()
            time.sleep(0.0005)
        job.cancel()
        st = job.wait(check=False)
        assert st["state"] == "FAILED" and st["error"] == TAD_ERR_CANCELLED, st
        st_q = q.wait()
        assert st_q["state"] == "COMPLETED"
        rows_q = q.result()
        q.release()
        # the cancel takes effect once the job running in the fit's place has ended
        assert t_job + st["total_ms"] * 1e-3 >= t_q + st_q["total_ms"] * 1e-3 - 0.002
    finally:
        eng.set_fit_sharing(0)
        job.release()
        cols.free()
    after = _solo(eng, small, "ARIMA", emit_all=True)[0]
    assert_same_rows(after, before, what="ARIMA after a cancel while parked")
    assert_same_rows(rows_q, ref_q, what="EWMA run while the fit was parked")


def test_budget_reserve_and_passes(eng):
    budget = 150 * MB + 64 * MB
    arima_t = _host_table([(20_000, 100, 17)])
    small_t = _host_table([(2_000, 100, 18)])
    big_t = _host_table([(1, 600_000, 19)])           # one connection: its 1/64 hash range does not fit 64 MiB
    eng.set_memory_budget(budget)
    try:
        ref_a = eng.run(arima_t, algo="ARIMA", tad_id="ref", emit_all=True)[0]
        ref_s = eng.run(small_t, algo="EWMA", tad_id="ref")[0]
        ref_b = eng.run(big_t, algo="EWMA", tad_id="ref")[0]
        ca, cs, cb = (eng.columns_from_numpy(t) for t in (arima_t, small_t, big_t))
        eng.set_fit_sharing(64 * MB)
        job = eng.submit(ca, algo="ARIMA", tad_id="passes", emit_all=True)
        _wait_fitting(job)
        t_big = time.time()
        qb = eng.submit(cb, algo="EWMA", tad_id="too-big")
        qs = eng.submit(cs, algo="EWMA", tad_id="fits")
        st_s = qs.wait()
        mem_s = qs.memory()
        rows_s = qs.result()
        st = job.wait()
        t_arima_done = time.time()
        mem_a, y, rows_a = job.memory(), job.yields(), job.result()
        st_b = qb.wait()
        rows_b = qb.result()
        for h in (job, qs, qb):
            h.release()
        for c in (ca, cs, cb):
            c.free()
    finally:
        eng.set_fit_sharing(0)
        eng.set_memory_budget(0)
    print("budget %d MiB: ARIMA %d passes, peak %.1f MiB, %d yields; EWMA beside it peak %.1f MiB; the large job "
          "finished %.2f s after the ARIMA job" % (budget >> 20, mem_a["passes"], mem_a["peak_workspace_bytes"] / MB,
                                                   y["yields"], mem_s["peak_workspace_bytes"] / MB,
                                                   t_big + st_b["total_ms"] * 1e-3 - t_arima_done))
    assert mem_a["passes"] >= 2 and y["yields"] >= 1
    assert mem_a["peak_workspace_bytes"] <= budget - 64 * MB
    assert mem_s["peak_workspace_bytes"] <= 64 * MB
    assert t_big + st_b["total_ms"] * 1e-3 >= t_arima_done - 0.005
    assert_same_rows(rows_a, ref_a, what="ARIMA in passes beside other jobs")
    assert_same_rows(rows_s, ref_s, what="EWMA in the reserve")
    assert_same_rows(rows_b, ref_b, what="EWMA too large for the reserve")


def test_sharing_off_keeps_the_order(eng):
    arima_cols = _device_table([(50_000, 100, 11)])
    ewma_cols = _device_table([(2_000, 100, 13)])
    job = eng.submit(arima_cols, algo="ARIMA", tad_id="off")
    try:
        _wait_fitting(job)
        time.sleep(0.5)
        q = eng.submit(ewma_cols, algo="EWMA", tad_id="behind")
        q.wait()
        assert job.poll()["state"] == "COMPLETED"
        q.release()
        job.wait()
        assert job.yields()["yields"] == 0
    finally:
        job.release()


@pytest.mark.parametrize("shape", ["long table", "long series"])
def test_steady_stream_keeps_the_fit_bound(eng, long_arima, shape):
    """EWMA jobs back to back for the whole fit phase: every yield waits until the fits the last one dropped have been
    fitted again, so no fit is dropped twice and the fit phase (parked time left out) stays within twice its solo time."""
    import threading
    if shape == "long table":
        cols, ref, st_ref = long_arima[0], long_arima[1], long_arima[2]
    else:
        cols = _device_table([(2_000, 100, 15), (1, 1_000, 16)])
        ref, st_ref, _ = _solo(eng, cols, "ARIMA", emit_all=True)
    ewma_cols = _device_table([(2_000, 100, 13)])
    ref_e = _solo(eng, ewma_cols, "EWMA")[0]
    eng.set_fit_sharing(RESERVE)
    job = eng.submit(cols, algo="ARIMA", tad_id="stream", emit_all=True)
    stop, got, errors = threading.Event(), [], []

    def stream():
        try:
            while not stop.is_set():
                q = eng.submit(ewma_cols, algo="EWMA", tad_id="stream")
                q.wait()
                if len(got) < 3:
                    got.append(q.result())
                q.release()
        except Exception as e:          # reported below
            errors.append(e)
    try:
        _wait_fitting(job)
        th = threading.Thread(target=stream)
        th.start()
        st = job.wait()
        stop.set()
        th.join()
        rows, y = job.result(), job.yields()
    finally:
        stop.set()
        eng.set_fit_sharing(0)
        job.release()
    solo = st_ref["phase_ms"]["detect"]
    print("steady stream, %s: detect %.0f ms (solo %.0f ms), %d yields, parked %.0f ms"
          % (shape, st["phase_ms"]["detect"], solo, y["yields"], y["parked_ms"]))
    assert not errors, errors
    assert y["yields"] >= 2
    assert st["phase_ms"]["detect"] <= 2.0 * solo
    assert_same_rows(rows, ref, what="ARIMA under a steady stream (%s)" % shape)
    for g in got:
        assert_same_rows(g, ref_e, what="EWMA of the stream")
