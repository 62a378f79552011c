"""Fitting beside a fit (TAD_FLAG_FIT_BESIDE): a flagged ARIMA job B queued behind a running ARIMA fit A runs in A's
yield, its fit in one launch with the rest of A's, and completes while A still fits.  Every job's rows, and every ARIMA
job's fit counts, equal those of a solo run."""
import time

import numpy as np
import pytest

from tests.test_gpu_fit_sharing import (LONG_SERIES, MB, RESERVE, TAD_ERR_CANCELLED, _device_table, _host_table, _solo,
                                        _wait_fitting)
from tests.util import assert_same_rows

pytestmark = pytest.mark.gpu

INTO_FIT_S = 0.5             # B is submitted this long into A's fit


@pytest.fixture(scope="module")
def eng():
    from theia_b200.engine import TadEngine
    e = TadEngine(device=0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def long_a(eng):
    """A: the 1.5e5 x 100 noisy table of tests/test_gpu_fit_sharing.py and its solo run."""
    cols = _device_table([(LONG_SERIES, 100, 14)])
    rows, st, p = _solo(eng, cols, "ARIMA", emit_all=True)
    return cols, rows, st, p


def _b(eng, series=2_000, seed=21):
    """B: a short ARIMA table and its solo run (rows, status, progress)."""
    cols = _device_table([(series, 100, seed)])
    rows, st, p = _solo(eng, cols, "ARIMA", emit_all=True)
    return cols, rows, st, p


def _same(job, ref, what):
    rows, p = job.result(), job.progress()
    assert_same_rows(rows, ref[1], what=what)
    assert (p["fits_done"], p["fits_total"]) == (ref[3]["fits_done"], ref[3]["fits_total"]), what


def _start_a(eng, a, reserve=RESERVE):
    eng.set_fit_sharing(reserve)
    job = eng.submit(a[0], algo="ARIMA", tad_id="A", emit_all=True)
    _wait_fitting(job)
    time.sleep(INTO_FIT_S)
    return job


def _wait_b_fitting(q, timeout=30.0):
    t0 = time.time()
    while q.progress()["fits_done"] == 0:
        assert q.poll()["state"] in ("SCHEDULED", "RUNNING"), q.poll()
        assert time.time() - t0 < timeout, "B did not start fitting"
        time.sleep(0.001)


def test_pairing(eng, long_a):
    b = _b(eng)
    solo_s = b[2]["total_ms"] * 1e-3
    job = _start_a(eng, long_a)
    samples = []
    try:
        t0 = time.time()
        q = eng.submit(b[0], algo="ARIMA", tad_id="B", emit_all=True, fit_beside=True)
        while q.poll()["state"] not in ("COMPLETED", "FAILED"):
            if q.poll()["state"] == "RUNNING":
                samples.append((job.progress()["fits_done"], q.progress()["fits_done"]))
            time.sleep(0.002)
        dt = time.time() - t0
        state_a = job.poll()["state"]
        q.wait()
        _same(q, b, "B beside A")
        yb = q.yields()
        q.release()
        job.wait()
        ya = job.yields()
        _same(job, long_a, "A with B beside it")
    finally:
        eng.set_fit_sharing(0)
        job.release()
    print("B beside A: %.3f s (solo %.3f s); A yields %d, parked %.1f ms; B yields %d"
          % (dt, solo_s, ya["yields"], ya["parked_ms"], yb["yields"]))
    assert state_a == "RUNNING"
    assert dt <= 3.0 * solo_s + 0.5
    assert ya["yields"] >= 1
    a_done = [s[0] for s in samples]
    b_done = [s[1] for s in samples if s[1] > 0]
    assert len(set(a_done)) >= 2, samples[:5]          # A's count moves while B runs
    assert len(set(b_done)) >= 1 and max(b_done) > 0


def test_no_flag_waits(eng, long_a):
    b = _b(eng)
    job = _start_a(eng, long_a)
    try:
        q = eng.submit(b[0], algo="ARIMA", tad_id="B-unflagged", emit_all=True)
        q.wait()
        assert job.poll()["state"] == "COMPLETED"
        _same(q, b, "unflagged B")
        q.release()
    finally:
        eng.set_fit_sharing(0)
        job.release()


def test_ewma_during_the_joint_fit(eng, long_a):
    b = _b(eng, series=8_000, seed=22)
    ewma_cols = _device_table([(2_000, 100, 13)])
    ref_e = _solo(eng, ewma_cols, "EWMA")[0]
    job = _start_a(eng, long_a)
    try:
        q = eng.submit(b[0], algo="ARIMA", tad_id="B", emit_all=True, fit_beside=True)
        _wait_b_fitting(q)
        t0 = time.time()
        e = eng.submit(ewma_cols, algo="EWMA", tad_id="E")
        e.wait()
        dt = time.time() - t0
        rows_e = e.result()
        e.release()
        q.wait()
        _same(q, b, "B with an EWMA job in its yield")
        yb = q.yields()
        q.release()
        job.wait()
        _same(job, long_a, "A with B and an EWMA job beside it")
    finally:
        eng.set_fit_sharing(0)
        job.release()
    print("EWMA during the joint fit: %.1f ms; B yields %d, parked %.1f ms" % (dt * 1e3, yb["yields"], yb["parked_ms"]))
    assert dt < 1.0
    assert yb["yields"] >= 1
    assert_same_rows(rows_e, ref_e, what="EWMA in B's yield")


def test_cancel_b(eng, long_a):
    b = _b(eng, series=8_000, seed=22)
    job = _start_a(eng, long_a)
    try:
        q = eng.submit(b[0], algo="ARIMA", tad_id="B", emit_all=True, fit_beside=True)
        _wait_b_fitting(q)
        q.cancel()
        st = q.wait(check=False)
        assert st["state"] == "FAILED" and st["error"] == TAD_ERR_CANCELLED, st
        q.release()
        job.wait()
        _same(job, long_a, "A after B was cancelled")
    finally:
        eng.set_fit_sharing(0)
        job.release()
    again = _solo(eng, b[0], "ARIMA", emit_all=True)[0]        # the context stays usable
    assert_same_rows(again, b[1], what="ARIMA after B was cancelled")


def test_cancel_a(eng, long_a):
    b = _b(eng, series=8_000, seed=22)
    job = _start_a(eng, long_a)
    try:
        q = eng.submit(b[0], algo="ARIMA", tad_id="B", emit_all=True, fit_beside=True)
        _wait_b_fitting(q)
        job.cancel()
        q.wait()
        _same(q, b, "B after A was cancelled")
        q.release()
        st = job.wait(check=False)
        assert st["state"] == "FAILED" and st["error"] == TAD_ERR_CANCELLED, st
    finally:
        eng.set_fit_sharing(0)
        job.release()
    again = _solo(eng, b[0], "ARIMA", emit_all=True)[0]        # the context stays usable
    assert_same_rows(again, b[1], what="ARIMA after A was cancelled beside it")


def test_b_in_passes_and_b_too_large(eng, long_a):
    b_t = _host_table([(20_000, 100, 23)])                 # 2e6 rows: passes inside half the reserve
    one = _host_table([(1, 100, 24)])
    big_t = {k: np.repeat(v, 20_000) for k, v in one.items()}   # one connection, 2e6 rows reduced to 100 points
    cb, cbig = eng.columns_from_numpy(b_t), eng.columns_from_numpy(big_t)
    try:
        ref_b = (cb,) + _solo(eng, cb, "ARIMA", emit_all=True)
        ref_big = (cbig,) + _solo(eng, cbig, "ARIMA", emit_all=True)
        job = _start_a(eng, long_a)
        try:
            q = eng.submit(cb, algo="ARIMA", tad_id="B-passes", emit_all=True, fit_beside=True)
            q.wait()
            state_a = job.poll()["state"]
            mem = q.memory()
            _same(q, ref_b, "B in passes")
            q.release()
            t_big = time.time()
            qb = eng.submit(cbig, algo="ARIMA", tad_id="B-too-large", emit_all=True, fit_beside=True)
            job.wait()
            t_a = time.time()
            st_big = qb.wait()
            _same(qb, ref_big, "B too large for half the reserve")
            qb.release()
            _same(job, long_a, "A with B in passes beside it")
        finally:
            eng.set_fit_sharing(0)
            job.release()
    finally:
        cb.free()
        cbig.free()
    print("B in passes: %d passes, peak %.1f MiB (half the reserve %d MiB)"
          % (mem["passes"], mem["peak_workspace_bytes"] / MB, RESERVE // 2 // MB))
    assert state_a == "RUNNING"
    assert mem["passes"] >= 2
    assert mem["peak_workspace_bytes"] <= RESERVE // 2
    assert t_big + st_big["total_ms"] * 1e-3 >= t_a - 0.005      # it ran after A


def test_two_partners_in_turn(eng, long_a):
    b, c = _b(eng), _b(eng, seed=25)
    job = _start_a(eng, long_a)
    done = {}
    try:
        t0 = time.time()
        qb = eng.submit(b[0], algo="ARIMA", tad_id="B", emit_all=True, fit_beside=True)
        qc = eng.submit(c[0], algo="ARIMA", tad_id="C", emit_all=True, fit_beside=True)
        for name, q in (("B", qb), ("C", qc)):
            st = q.wait()
            done[name] = t0 + st["total_ms"] * 1e-3
        state_a = job.poll()["state"]
        _same(qb, b, "B, the first partner")
        _same(qc, c, "C, the second partner")
        for q in (qb, qc):
            q.release()
        job.wait()
        _same(job, long_a, "A with two partners")
    finally:
        eng.set_fit_sharing(0)
        job.release()
    print("two partners: B done %.3f s, C done %.3f s after submission" % (done["B"] - t0, done["C"] - t0))
    assert state_a == "RUNNING"
    assert done["B"] < done["C"]


def test_small_reserve_does_not_pair(eng, long_a):
    b = _b(eng)
    job = _start_a(eng, long_a, reserve=127 * MB)
    try:
        q = eng.submit(b[0], algo="ARIMA", tad_id="B-small-reserve", emit_all=True, fit_beside=True)
        q.wait()
        assert job.poll()["state"] == "COMPLETED"
        _same(q, b, "B behind A with a small reserve")
        q.release()
    finally:
        eng.set_fit_sharing(0)
        job.release()


def test_long_series_in_a(eng):
    """A's fit is down to one 1,000-point connection when B arrives: the fits A's yield dropped are fitted again in the
    joint launch before it ends, so none is dropped twice, and A's counts equal its solo counts."""
    a_cols = _device_table([(2_000, 100, 15), (1, 1_000, 16)])
    a = (a_cols,) + _solo(eng, a_cols, "ARIMA", emit_all=True)
    b = _b(eng)
    eng.set_fit_sharing(RESERVE)
    job = eng.submit(a_cols, algo="ARIMA", tad_id="A-long-series", emit_all=True)
    try:
        _wait_fitting(job)
        time.sleep(1.0)                          # the short series are done: only the long one is being fitted
        q = eng.submit(b[0], algo="ARIMA", tad_id="B", emit_all=True, fit_beside=True)
        q.wait()
        state_a = job.poll()["state"]
        _same(q, b, "B beside one long series")
        q.release()
        job.wait()
        _same(job, a, "A with one long series")
    finally:
        eng.set_fit_sharing(0)
        job.release()
    assert state_a == "RUNNING"
