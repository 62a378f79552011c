"""A streamed ARIMA job fitting beside a running fit (TAD_FLAG_SHARE | TAD_FLAG_FIT_BESIDE on a streamed job): it runs
in the yield of the fit, its passes each in one launch with the rest of that fit, and completes while the fit still
runs; the reverse pairing, a job fitting beside a streamed fit, too.  Every job's rows, and every ARIMA job's fit counts
and text names, equal those of a solo run of the same job."""
import threading
import time

import numpy as np
import pytest

from tests.test_gpu_fit_beside import _wait_b_fitting
from tests.test_gpu_fit_sharing import (LONG_SERIES, MB, RESERVE, TAD_ERR_CANCELLED, _device_table, _host_table, _solo,
                                        _wait_fitting)
from tests.test_gpu_fit_sharing_stream import (ARIMA_BUDGET, HOST, LONG_POINTS, Feeder, check_arima, feed,  # noqa: F401
                                               long_stream, names_of, same_names, stream_solo, text_blocks)
from tests.util import assert_same_rows

pytestmark = pytest.mark.gpu

INTO_FIT_S = 0.5             # B is submitted this long into A's fit
FINISHED = ("COMPLETED", "FAILED")
PASSES_N = 20_000            # B in passes: 2e6 rows, at least 2 passes in half the reserve
MID_SERIES = 50_000          # a streamed A shorter than the long table: 5e6 rows in passes under MID_BUDGET
MID_BUDGET = 512 * MB


@pytest.fixture(scope="module")
def eng():
    from theia_b200.engine import TadEngine
    e = TadEngine(device=0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def long_a(eng):
    """A: the 1.5e5 x 100 noisy table on the device and its solo tad_submit ARIMA run."""
    cols = _device_table([(LONG_SERIES, 100, 14)])
    rows, st, p = _solo(eng, cols, "ARIMA", emit_all=True)
    return cols, rows, st, p


def _stream_b(eng, series, seed):
    """A streamed B: `series` x 100 points in host blocks with text addresses, and its solo run."""
    blocks = text_blocks(_host_table([(series, 100, seed)]))
    return blocks, stream_solo(eng, blocks, "ARIMA", emit_all=True)


@pytest.fixture(scope="module")
def b_small(eng):
    return _stream_b(eng, 2_000, 21)


@pytest.fixture(scope="module")
def b_long(eng):
    """A B whose fit lasts long enough to act on while it runs."""
    return _stream_b(eng, 8_000, 22)


@pytest.fixture(scope="module")
def b_passes(eng):
    """A B of 2e6 rows and its solo run in half the reserve, without a host store: (blocks, ref, solo rounds)."""
    blocks = text_blocks(_host_table([(PASSES_N, 100, 23)]))
    eng.set_memory_budget(RESERVE // 2)
    job = eng.submit_stream(algo="ARIMA", tad_id="solo", emit_all=True, rows_hint=PASSES_N * 100)
    try:
        rounds = feed(job, blocks)
        st = job.wait()
        ref = (job.result(), st, job.progress(), names_of(job), job.memory())
    finally:
        job.release()
        eng.set_memory_budget(0)
    assert ref[4]["passes"] >= 2 and rounds >= 2
    return blocks, ref, rounds


def _start_a(eng, a, reserve=RESERVE):
    eng.set_fit_sharing(reserve)
    job = eng.submit(a[0], algo="ARIMA", tad_id="A", emit_all=True)
    _wait_fitting(job)
    time.sleep(INTO_FIT_S)
    return job


def _same(job, ref, what):
    """A tad_submit job's rows and fit counts against its solo (rows, status, progress)."""
    assert_same_rows(job.result(), ref[1], what=what)
    p = job.progress()
    assert (p["fits_done"], p["fits_total"]) == (ref[3]["fits_done"], ref[3]["fits_total"]), what


def _submit_b(eng, blocks, tad_id="B", **kw):
    args = dict(share=True, fit_beside=True)
    args.update(kw)
    q = eng.submit_stream(algo="ARIMA", tad_id=tad_id, emit_all=True, **args)
    fd = Feeder(q, blocks)
    fd.start()
    return q, fd


def _finish(eng, *jobs_and_feeders):
    """Cleanup: a failed check must not leave a feeder waiting."""
    for job, fd in jobs_and_feeders:
        if job is not None and job.h:
            job.cancel()
        if fd is not None:
            fd.join()
        if job is not None:
            job.release()
    eng.set_fit_sharing(0)
    eng.set_memory_budget(0)
    eng.set_host_budget(0)


def _runs_after(eng, b):
    """The context runs a further job correctly."""
    blocks, ref = b
    after = stream_solo(eng, blocks, "ARIMA", emit_all=True)
    assert_same_rows(after[0], ref[0], what="a streamed ARIMA job after the case")
    same_names(after[3], ref[3], "a streamed ARIMA job after the case")


def test_streamed_b_beside_submitted_a(eng, long_a, b_small):
    blocks, ref = b_small
    solo_s = ref[1]["total_ms"] * 1e-3
    job = _start_a(eng, long_a)
    q = fd = None
    samples = []
    try:
        t0 = time.time()
        q, fd = _submit_b(eng, blocks)
        while q.poll()["state"] not in FINISHED:
            if q.poll()["state"] == "RUNNING":
                samples.append((job.progress()["fits_done"], q.progress()["fits_done"]))
            time.sleep(0.002)
        dt = time.time() - t0
        state_a = job.poll()["state"]
        fd.join()
        assert fd.error is None, fd.error
        _, yb, _ = check_arima(q, ref, "streamed B beside A")
        job.wait()
        ya = job.yields()
        _same(job, long_a, "A with a streamed B beside it")
    finally:
        _finish(eng, (q, fd), (job, None))
    print("streamed B beside A: %.3f s (solo %.3f s); A yields %d, parked %.1f ms; B yields %d"
          % (dt, solo_s, ya["yields"], ya["parked_ms"], yb["yields"]))
    assert state_a == "RUNNING"
    assert dt <= 3.0 * solo_s + 0.5
    assert ya["yields"] >= 1
    a_done = [s[0] for s in samples]
    b_done = [s[1] for s in samples if s[1] > 0]
    assert len(set(a_done)) >= 2, samples[:5]          # A's count moves while B runs
    assert len(set(b_done)) >= 1 and max(b_done) > 0


@pytest.mark.parametrize("host", [0, HOST])
def test_submitted_b_beside_streamed_a(eng, long_stream, host):
    blocks, ref = long_stream
    b_cols = _device_table([(2_000, 100, 21)])
    ref_b = _solo(eng, b_cols, "ARIMA", emit_all=True)
    eng.set_memory_budget(ARIMA_BUDGET)
    eng.set_host_budget(host)
    eng.set_fit_sharing(RESERVE)
    job = eng.submit_stream(algo="ARIMA", tad_id="A", share=True, rows_hint=LONG_SERIES * 100 + LONG_POINTS)
    fd = Feeder(job, blocks)
    fd.start()
    q = None
    try:
        _wait_fitting(job)
        time.sleep(INTO_FIT_S)
        q = eng.submit(b_cols, algo="ARIMA", tad_id="B", emit_all=True, fit_beside=True)
        q.wait()
        state_a = job.poll()["state"]
        _same(q, (None,) + ref_b, "B beside a streamed A")
        fd.join()
        assert fd.error is None, fd.error
        _, y, mem = check_arima(job, ref, "streamed A with B beside it")
    finally:
        _finish(eng, (q, None), (job, fd))
    print("host %d: B beside the streamed fit; A %d passes, %d rounds, %d yields, parked %.1f ms, stored %d rows"
          % (host, mem["passes"], fd.rounds, y["yields"], y["parked_ms"], mem["stored_rows"]))
    assert state_a == "RUNNING"
    assert y["yields"] >= 1
    assert mem["peak_workspace_bytes"] <= ARIMA_BUDGET - RESERVE
    assert (mem["stored_rows"] > 0) == (host > 0)


def test_both_streamed_with_text_keys(eng, b_small):
    """A streamed A of 5e6 rows in passes from the host store (512 MiB budget less the reserve) and a streamed B, each
    with its own dictionaries."""
    blocks = text_blocks(_host_table([(MID_SERIES, 100, 25)]))
    ref = stream_solo(eng, blocks, "ARIMA", budget=MID_BUDGET, host=HOST, rows_hint=MID_SERIES * 100)
    b_blocks, ref_b = b_small
    eng.set_memory_budget(MID_BUDGET)
    eng.set_host_budget(HOST)
    eng.set_fit_sharing(RESERVE)
    job = eng.submit_stream(algo="ARIMA", tad_id="A", share=True, rows_hint=MID_SERIES * 100)
    fd = Feeder(job, blocks)
    fd.start()
    q = fb = None
    try:
        _wait_fitting(job)
        time.sleep(INTO_FIT_S)
        q, fb = _submit_b(eng, b_blocks)
        fb.join()
        assert fb.error is None, fb.error
        q.wait()
        state_a = job.poll()["state"]
        check_arima(q, ref_b, "streamed B beside a streamed A")
        fd.join()
        assert fd.error is None, fd.error
        _, y, mem = check_arima(job, ref, "streamed A with a streamed B beside it")
    finally:
        _finish(eng, (q, fb), (job, fd))
    print("both streamed: A %d passes, stored %d rows, %d yields" % (mem["passes"], mem["stored_rows"], y["yields"]))
    assert state_a == "RUNNING"
    assert y["yields"] >= 1
    assert mem["passes"] >= 2 and mem["stored_rows"] > 0


def test_one_flag_alone_waits(eng, long_a, b_small):
    """A streamed ARIMA B with TAD_FLAG_SHARE only, and one with TAD_FLAG_FIT_BESIDE only, wait for A's fit phase."""
    blocks, ref = b_small
    job = _start_a(eng, long_a)
    q1 = f1 = q2 = f2 = None
    try:
        q1, f1 = _submit_b(eng, blocks, tad_id="B-share", fit_beside=False)
        q2, f2 = _submit_b(eng, blocks, tad_id="B-beside", share=False)
        states = []
        for q, fd, what in ((q1, f1, "TAD_FLAG_SHARE alone"), (q2, f2, "TAD_FLAG_FIT_BESIDE alone")):
            q.wait()
            states.append(job.poll()["state"])
            fd.join()
            assert fd.error is None, fd.error
            check_arima(q, ref, what)
        job.wait()
        y = job.yields()
        _same(job, long_a, "A with one-flag jobs queued")
    finally:
        _finish(eng, (q1, f1), (q2, f2), (job, None))
    assert states == ["COMPLETED", "COMPLETED"]
    assert y["yields"] == 0


def test_unfed_b_does_not_park_the_fit(eng, long_a, b_small):
    blocks, ref = b_small
    job = _start_a(eng, long_a)
    q = fd = None
    try:
        q = eng.submit_stream(algo="ARIMA", tad_id="B-unfed", emit_all=True, share=True, fit_beside=True)
        time.sleep(1.0)
        state_q = q.poll()["state"]
        fd = Feeder(q, blocks)
        fd.start()
        fd.join()
        assert fd.error is None, fd.error
        q.wait()
        state_a = job.poll()["state"]
        check_arima(q, ref, "streamed B fed late")
        job.wait()
        y = job.yields()
        _same(job, long_a, "A with a streamed B fed late")
    finally:
        _finish(eng, (q, fd), (job, None))
    assert state_q == "SCHEDULED"
    assert state_a == "RUNNING"
    assert y["yields"] == 1            # the fed job's yield only: the second it waited unfed made none


@pytest.mark.parametrize("host", [0, HOST])
def test_b_in_passes(eng, long_a, b_passes, host):
    """Without a host store B's caller delivers as many rounds as alone, A parked meanwhile; with one, B is delivered
    once."""
    blocks, ref, solo_rounds = b_passes
    eng.set_host_budget(host)          # before A: A's start sets the store's page size, which B's store shares
    job = _start_a(eng, long_a)
    q = fd = None
    try:
        q, fd = _submit_b(eng, blocks, rows_hint=PASSES_N * 100)
        fd.join()
        assert fd.error is None, fd.error
        q.wait()
        state_a = job.poll()["state"]
        _, _, mem = check_arima(q, ref, "streamed B in passes beside A")
        job.wait()
        _same(job, long_a, "A with a streamed B in passes beside it")
    finally:
        _finish(eng, (q, fd), (job, None))
    print("host %d: B %d passes, %d rounds (solo %d), stored %d rows, peak %.1f MiB"
          % (host, mem["passes"], fd.rounds, solo_rounds, mem["stored_rows"], mem["peak_workspace_bytes"] / MB))
    assert state_a == "RUNNING"
    assert mem["passes"] >= 2
    assert mem["peak_workspace_bytes"] <= RESERVE // 2
    if host:
        assert fd.rounds == 1 and mem["stored_rows"] > 0
    else:
        assert fd.rounds == solo_rounds and mem["stored_rows"] == 0


def test_b_too_large_for_half_the_reserve(eng, long_a):
    """One connection of 2e6 rows: its 1/64 hash range does not fit half a 128 MiB reserve."""
    one = _host_table([(1, 100, 24)])
    big = {k: np.repeat(v, 20_000) for k, v in one.items()}
    blocks = [({k: v[lo:lo + 65_536] for k, v in big.items()}, None) for lo in range(0, len(big["flow_end"]), 65_536)]
    ref = stream_solo(eng, blocks, "ARIMA", emit_all=True)
    job = _start_a(eng, long_a, reserve=128 * MB)
    q = fd = None
    try:
        q = eng.submit_stream(algo="ARIMA", tad_id="B-too-large", emit_all=True, share=True, fit_beside=True)
        for b, _ in blocks:
            q.push(b)
        again = q.end()
        t0 = time.time()
        while q.poll()["state"] == "RUNNING" and time.time() - t0 < 1.0:     # the round closes just before the put-back
            time.sleep(0.001)
        st_q, p_q = q.poll(), q.progress()
        fd = Feeder(q, blocks)
        fd.start()
        q.wait()
        state_a = job.poll()["state"]
        fd.join()
        assert fd.error is None, fd.error
        assert_same_rows(q.result(), ref[0], what="streamed B too large for half the reserve")
        p = q.progress()
        assert (p["fits_done"], p["fits_total"]) == (ref[2]["fits_done"], ref[2]["fits_total"])
        job.wait()
        y = job.yields()
        _same(job, long_a, "A with a streamed B too large for half the reserve")
    finally:
        _finish(eng, (q, fd), (job, None))
    assert again
    assert st_q["state"] == "SCHEDULED" and st_q["completed_stages"] == 0
    assert p_q == {"passes_done": 0, "passes": 0, "fits_done": 0, "fits_total": 0}
    assert state_a == "COMPLETED"      # it ran in its turn, after A
    assert y["yields"] >= 1


def test_inner_yield(eng, long_a, b_long):
    """A fed, flagged streamed EWMA job submitted during the joint fit runs in B's yield (A's and B's dictionaries
    parked) and completes before B."""
    blocks, ref = b_long
    e_blocks = text_blocks(_host_table([(2_000, 100, 13)]), block=8_192)
    ref_e = stream_solo(eng, e_blocks, "EWMA")
    job = _start_a(eng, long_a)
    q = fd = e = fe = None
    try:
        q, fd = _submit_b(eng, blocks)
        _wait_b_fitting(q)
        t0 = time.time()
        e = eng.submit_stream(algo="EWMA", tad_id="E", share=True)
        fe = Feeder(e, e_blocks)
        fe.start()
        fe.join()
        e.wait()
        dt = time.time() - t0
        state_b = q.poll()["state"]
        assert fe.error is None, fe.error
        assert_same_rows(e.result(), ref_e[0], what="streamed EWMA in B's yield")
        same_names(names_of(e), ref_e[3], "streamed EWMA in B's yield")
        fd.join()
        assert fd.error is None, fd.error
        _, yb, _ = check_arima(q, ref, "streamed B with an EWMA job in its yield")
        job.wait()
        _same(job, long_a, "A with B and an EWMA job beside it")
    finally:
        _finish(eng, (e, fe), (q, fd), (job, None))
    print("EWMA in B's yield: %.1f ms; B yields %d, parked %.1f ms" % (dt * 1e3, yb["yields"], yb["parked_ms"]))
    assert state_b == "RUNNING"
    assert yb["yields"] >= 1


def test_cancel_b_during_its_fit(eng, long_a, b_long, b_small):
    blocks, _ = b_long
    job = _start_a(eng, long_a)
    q = fd = None
    try:
        q, fd = _submit_b(eng, blocks)
        _wait_b_fitting(q)
        q.cancel()
        st = q.wait(check=False)
        state_a = job.poll()["state"]
        fd.join()
        job.wait()
        _same(job, long_a, "A after a streamed B was cancelled")
    finally:
        _finish(eng, (q, fd), (job, None))
    assert st["state"] == "FAILED" and st["error"] == TAD_ERR_CANCELLED, st
    assert fd.error is not None and fd.error.code == TAD_ERR_CANCELLED, fd.error
    assert state_a == "RUNNING"
    _runs_after(eng, b_small)


class RoundFeeder(threading.Thread):
    """Feeds one round, then waits for `go` before the next; `error` holds what a push or end call raised."""

    def __init__(self, job, blocks):
        super().__init__()
        self.job, self.blocks, self.error = job, blocks, None
        self.between, self.go = threading.Event(), threading.Event()

    def run(self):
        try:
            for b, txt in self.blocks:
                self.job.push(b, text=txt)
            assert self.job.end()
            self.between.set()
            self.go.wait()
            for b, txt in self.blocks:
                self.job.push(b, text=txt)
            self.job.end()
        except Exception as e:          # checked by the test
            self.error = e


def test_cancel_b_between_rounds(eng, long_a, b_passes, b_small):
    blocks = b_passes[0]
    job = _start_a(eng, long_a)
    q = fd = None
    try:
        q = eng.submit_stream(algo="ARIMA", tad_id="B", emit_all=True, share=True, fit_beside=True,
                              rows_hint=PASSES_N * 100)
        fd = RoundFeeder(q, blocks)
        fd.start()
        assert fd.between.wait(120.0), fd.error
        q.cancel()
        st = q.wait(check=False)
        state_a = job.poll()["state"]
        fd.go.set()
        fd.join()
        job.wait()
        _same(job, long_a, "A after a streamed B was cancelled between rounds")
    finally:
        if fd is not None:
            fd.go.set()
        _finish(eng, (q, fd), (job, None))
    assert st["state"] == "FAILED" and st["error"] == TAD_ERR_CANCELLED, st
    assert fd.error is not None and getattr(fd.error, "code", None) == TAD_ERR_CANCELLED, fd.error
    assert state_a == "RUNNING"
    _runs_after(eng, b_small)


def test_cancel_a_beside_streamed_b(eng, long_a, b_long, b_small):
    blocks, ref = b_long
    job = _start_a(eng, long_a)
    q = fd = None
    try:
        q, fd = _submit_b(eng, blocks)
        _wait_b_fitting(q)
        job.cancel()
        while True:
            state_a = job.poll()["state"]       # read before B's: A fails only once B has ended
            if q.poll()["state"] in FINISHED:
                break
            assert state_a == "RUNNING"
            time.sleep(0.002)
        fd.join()
        assert fd.error is None, fd.error
        check_arima(q, ref, "streamed B after A was cancelled")
        st = job.wait(check=False)
    finally:
        _finish(eng, (q, fd), (job, None))
    assert st["state"] == "FAILED" and st["error"] == TAD_ERR_CANCELLED, st
    _runs_after(eng, b_small)
