"""Fit sharing for streamed jobs (TAD_FLAG_SHARE): a streamed ARIMA job's fit yields with its text key dictionaries, its
round and its host row store pages parked, and flagged streamed EWMA and DBSCAN jobs run in a fit's yields.  Every job's
rows, a text job's names and the ARIMA job's fit counts equal those of a solo run of the same job."""
import threading
import time

import numpy as np
import pytest

from theia_b200 import _lib as L
from theia_b200 import synth
from tests.util import assert_same_rows

from .test_text_keys import column_from_names, text_table

pytestmark = pytest.mark.gpu

TAD_ERR_CANCELLED = -6
MB = 1 << 20
RESERVE = 256 * MB
# the long table of tests/test_gpu_fit_sharing.py: its fit phase takes about 10 s on an H100
LONG_SERIES = 150_000
LONG_POINTS = 4_000
BLOCK = 65_536
ARIMA_BUDGET = 1536 * MB     # the long table's streamed ARIMA job runs in hash-range passes under it
HOST = 1 << 30               # room for the long table's rows (480 MB) and for an interleaved job's beside them


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


def _name(v: int) -> bytes:
    return b"fd00::%x" % v


def text_blocks(table, block=BLOCK):
    """The table in host blocks of `block` rows with both address slots as text (tad_stream_push_text)."""
    slots = {s: text_table(table[s], _name) for s in ("src_ip", "dst_ip")}
    n = len(table["flow_end"])
    out = []
    for lo in range(0, n, block):
        hi = min(n, lo + block)
        b = {k: v[lo:hi] for k, v in table.items()}
        b.update(src_ip=None, dst_ip=None)
        out.append((b, {s: column_from_names(names, inv[lo:hi]) for s, (names, inv) in slots.items()}))
    return out


def feed(job, blocks):
    """Every round of a streamed job until its input is complete; returns the number of rounds."""
    n, again = 0, True
    while again:
        for b, txt in blocks:
            job.push(b, text=txt)
        again = job.end()
        n += 1
    return n


class Feeder(threading.Thread):
    """A streamed job's feeding thread; `error` holds what its push or end call raised."""

    def __init__(self, job, blocks):
        super().__init__()
        self.job, self.blocks, self.error, self.rounds = job, blocks, None, 0

    def run(self):
        try:
            self.rounds = feed(self.job, self.blocks)
        except Exception as e:          # checked by the test
            self.error = e


def names_of(job):
    return {s: job.names(s) for s in ("src_ip", "dst_ip")}


def stream_solo(eng, blocks, algo, budget=0, host=0, **kw):
    """A streamed job alone on the context, sharing off: (rows, status, progress, names, memory)."""
    eng.set_memory_budget(budget)
    eng.set_host_budget(host)
    job = eng.submit_stream(algo=algo, tad_id="solo", **kw)
    try:
        feed(job, blocks)
        st = job.wait()
        return job.result(), st, job.progress(), names_of(job) if blocks[0][1] else None, job.memory()
    finally:
        job.release()
        eng.set_memory_budget(0)
        eng.set_host_budget(0)


def same_names(got, want, what):
    for s in ("src_ip", "dst_ip"):
        for a, b in zip(got[s], want[s]):
            assert np.array_equal(a, b), "%s: names of %s differ" % (what, s)


@pytest.fixture(scope="module")
def long_arima(eng):
    """The long table on the device and its solo tad_submit ARIMA run (sharing off)."""
    cols = _device_table([(LONG_SERIES, 100, 14)])
    rows, st, p = _solo(eng, cols, "ARIMA", emit_all=True)
    return cols, rows, st, p


@pytest.fixture(scope="module")
def long_stream(eng):
    """The long table (plus one 4,000-point connection) in host blocks with text addresses, and the solo run of its
    streamed ARIMA job in passes under ARIMA_BUDGET."""
    blocks = text_blocks(_host_table([(LONG_SERIES, 100, 14), (1, LONG_POINTS, 16)]))
    ref = stream_solo(eng, blocks, "ARIMA", budget=ARIMA_BUDGET, rows_hint=LONG_SERIES * 100 + LONG_POINTS)
    assert ref[4]["passes"] >= 2
    return blocks, ref


@pytest.fixture(scope="module")
def small_stream(eng):
    """A 2e5-row table in host blocks with text addresses, and its solo streamed EWMA run."""
    blocks = text_blocks(synth.make_flows(2_000, 100, seed=41), block=8_192)
    return blocks, stream_solo(eng, blocks, "EWMA")


def check_arima(job, ref, what):
    rows_ref, _, p_ref, names_ref, _ = ref
    st = job.wait()
    assert_same_rows(job.result(), rows_ref, what=what)
    p = job.progress()
    assert (p["fits_done"], p["fits_total"]) == (p_ref["fits_done"], p_ref["fits_total"]), what
    same_names(names_of(job), names_ref, what)
    return st, job.yields(), job.memory()


@pytest.mark.parametrize("host", [0, HOST])
def test_streamed_arima_yields(eng, long_stream, host):
    blocks, ref = long_stream
    ewma_cols = _device_table([(2_000, 100, 13)])
    ref_e = _solo(eng, ewma_cols, "EWMA")[0]
    eng.set_memory_budget(ARIMA_BUDGET)
    eng.set_host_budget(host)
    eng.set_fit_sharing(RESERVE)
    job = eng.submit_stream(algo="ARIMA", tad_id="long", share=True, rows_hint=LONG_SERIES * 100 + LONG_POINTS)
    fd = Feeder(job, blocks)
    fd.start()
    try:
        _wait_fitting(job)
        time.sleep(0.2)
        t0 = time.time()
        q = eng.submit(ewma_cols, algo="EWMA", tad_id="beside")
        q.wait()
        dt = time.time() - t0
        state = job.poll()["state"]
        rows_q = q.result()
        q.release()
        fd.join()
        assert fd.error is None, fd.error
        st, y, mem = check_arima(job, ref, "streamed ARIMA beside a job")
    finally:
        job.cancel()                    # a failed check must not leave the feeder waiting
        fd.join()
        eng.set_fit_sharing(0)
        eng.set_memory_budget(0)
        eng.set_host_budget(0)
        job.release()
    print("host %d: EWMA beside the streamed fit %.3f s; ARIMA %d passes, %d rounds, %d yields, parked %.1f ms, stored "
          "%d rows" % (host, dt, mem["passes"], fd.rounds, y["yields"], y["parked_ms"], mem["stored_rows"]))
    assert state == "RUNNING"
    assert dt < 1.0
    assert y["yields"] >= 1
    assert mem["peak_workspace_bytes"] <= ARIMA_BUDGET - RESERVE
    assert (mem["stored_rows"] > 0) == (host > 0)
    assert_same_rows(rows_q, ref_e, what="EWMA beside the streamed fit")


@pytest.mark.parametrize("algo,flt", [("EWMA", None), ("DBSCAN", None), ("EWMA", {"dst_ip": ("icontains", b"A")})])
def test_streamed_job_runs_in_a_yield(eng, long_arima, small_stream, algo, flt):
    """A flagged streamed job fed by its own thread beside a tad_submit ARIMA fit; the third case is an svc-style job
    (sums, a predicate on the service name) submitted with tad_submit_stream_filtered, its predicate on the GPU."""
    blocks = small_stream[0]
    kw = dict(text_filter=flt)
    if flt is not None:
        kw["reducer"] = L.TAD_REDUCE_SUM
    ref = small_stream[1] if (algo, flt) == ("EWMA", None) else stream_solo(eng, blocks, algo, **kw)
    eng.set_fit_sharing(RESERVE)
    job = eng.submit(long_arima[0], algo="ARIMA", tad_id="long", emit_all=True)
    try:
        _wait_fitting(job)
        time.sleep(0.2)
        t0 = time.time()
        q = eng.submit_stream(algo=algo, tad_id="beside", share=True, **kw)
        fd = Feeder(q, blocks)
        fd.start()
        fd.join()
        st_q = q.wait()
        dt = time.time() - t0
        state = job.poll()["state"]
        assert fd.error is None, fd.error
        rows_q, names_q = q.result(), names_of(q)
        q.release()
        job.wait()
        assert_same_rows(job.result(), long_arima[1], what="ARIMA beside a streamed job")
        p, p_ref = job.progress(), long_arima[3]
        assert (p["fits_done"], p["fits_total"]) == (p_ref["fits_done"], p_ref["fits_total"])
        y = job.yields()
    finally:
        eng.set_fit_sharing(0)
        job.release()
    print("streamed %s%s beside the fit: %.3f s (%d rounds, rows kept %d); ARIMA %d yields, parked %.1f ms"
          % (algo, " svc" if flt else "", dt, fd.rounds, st_q["rows_kept"], y["yields"], y["parked_ms"]))
    assert state == "RUNNING"
    assert y["yields"] >= 1
    assert_same_rows(rows_q, ref[0], what="streamed %s in a yield" % algo)
    same_names(names_q, ref[3], "streamed %s in a yield" % algo)


def test_both_streamed(eng, long_stream):
    """The parked ARIMA job holds dictionaries and store slabs; the streamed EWMA job run in its yield builds its own
    dictionaries and uses the store room left."""
    blocks, ref = long_stream
    reserve = 64 * MB
    ewma_blocks = text_blocks(synth.make_flows(20_000, 100, seed=42))        # 2e6 rows: passes in the reserve
    n_e = 20_000 * 100
    ref_e = stream_solo(eng, ewma_blocks, "EWMA", budget=reserve, host=HOST, rows_hint=n_e)
    assert ref_e[4]["passes"] >= 2 and ref_e[4]["stored_rows"] > 0
    eng.set_memory_budget(ARIMA_BUDGET)
    eng.set_host_budget(HOST)
    eng.set_fit_sharing(reserve)
    job = eng.submit_stream(algo="ARIMA", tad_id="long", share=True, rows_hint=LONG_SERIES * 100 + LONG_POINTS)
    fd = Feeder(job, blocks)
    fd.start()
    try:
        _wait_fitting(job)
        time.sleep(0.2)
        q = eng.submit_stream(algo="EWMA", tad_id="beside", share=True, rows_hint=n_e)
        fe = Feeder(q, ewma_blocks)
        fe.start()
        fe.join()
        q.wait()
        state = job.poll()["state"]
        assert fe.error is None, fe.error
        rows_q, names_q, mem_q = q.result(), names_of(q), q.memory()
        q.release()
        fd.join()
        assert fd.error is None, fd.error
        st, y, mem = check_arima(job, ref, "streamed ARIMA beside a streamed job")
    finally:
        job.cancel()                    # a failed check must not leave the feeder waiting
        fd.join()
        eng.set_fit_sharing(0)
        eng.set_memory_budget(0)
        eng.set_host_budget(0)
        job.release()
    print("both streamed: EWMA %d passes, %d rounds, stored %d rows, host peak %.0f MiB; ARIMA stored %d rows, host peak "
          "%.0f MiB, %d yields" % (mem_q["passes"], fe.rounds, mem_q["stored_rows"], mem_q["peak_host_bytes"] / MB,
                                   mem["stored_rows"], mem["peak_host_bytes"] / MB, y["yields"]))
    assert state == "RUNNING"
    assert y["yields"] >= 1
    assert mem["stored_rows"] > 0 and mem_q["stored_rows"] > 0
    assert mem_q["peak_workspace_bytes"] <= reserve
    assert mem_q["peak_host_bytes"] <= HOST
    assert_same_rows(rows_q, ref_e[0], what="streamed EWMA beside the streamed fit")
    same_names(names_q, ref_e[3], "streamed EWMA beside the streamed fit")


def test_no_flag_no_sharing(eng, long_arima, long_stream, small_stream):
    blocks, ref = long_stream
    ewma_cols = _device_table([(2_000, 100, 13)])
    eng.set_memory_budget(ARIMA_BUDGET)
    eng.set_fit_sharing(RESERVE)
    # a streamed ARIMA job without the flag does not yield
    job = eng.submit_stream(algo="ARIMA", tad_id="long", rows_hint=LONG_SERIES * 100 + LONG_POINTS)
    fd = Feeder(job, blocks)
    fd.start()
    try:
        _wait_fitting(job)
        time.sleep(0.2)
        q = eng.submit(ewma_cols, algo="EWMA", tad_id="behind")
        q.wait()
        assert job.poll()["state"] == "COMPLETED"
        q.release()
        fd.join()
        assert fd.error is None, fd.error
        _, y, _ = check_arima(job, ref, "streamed ARIMA without the flag")
    finally:
        job.cancel()                    # a failed check must not leave the feeder waiting
        fd.join()
        eng.set_memory_budget(0)
        job.release()
    assert y["yields"] == 0
    # a streamed EWMA job without the flag waits for the fit phase of a tad_submit ARIMA job
    job = eng.submit(long_arima[0], algo="ARIMA", tad_id="long", emit_all=True)
    try:
        _wait_fitting(job)
        time.sleep(0.2)
        q = eng.submit_stream(algo="EWMA", tad_id="behind")
        fe = Feeder(q, small_stream[0])
        fe.start()
        fe.join()
        assert fe.error is None, fe.error
        q.wait()
        assert job.poll()["state"] == "COMPLETED"
        assert_same_rows(q.result(), small_stream[1][0], what="streamed EWMA without the flag")
        q.release()
        job.wait()
        assert job.yields()["yields"] == 0
    finally:
        eng.set_fit_sharing(0)
        job.release()


def test_unfed_job_does_not_park_the_fit(eng, long_arima, small_stream):
    blocks, ref = small_stream
    eng.set_fit_sharing(RESERVE)
    job = eng.submit(long_arima[0], algo="ARIMA", tad_id="long", emit_all=True)
    try:
        _wait_fitting(job)
        q = eng.submit_stream(algo="EWMA", tad_id="unfed", share=True)
        time.sleep(1.0)
        assert q.poll()["state"] == "SCHEDULED"
        t0 = time.time()
        fd = Feeder(q, blocks)
        fd.start()
        fd.join()
        q.wait()
        dt = time.time() - t0
        assert fd.error is None, fd.error
        state = job.poll()["state"]
        rows_q = q.result()
        q.release()
        job.wait()
        y = job.yields()
    finally:
        eng.set_fit_sharing(0)
        job.release()
    print("unfed job: ran %.3f s after its feeder started; ARIMA %d yields" % (dt, y["yields"]))
    assert state == "RUNNING"
    assert y["yields"] == 1            # the fed job's yield only: the second the job waited unfed made none
    assert_same_rows(rows_q, ref[0], what="EWMA fed late")


def test_job_that_does_not_fit_the_reserve(eng, long_arima):
    """A flagged streamed job whose 1/64 hash range does not fit a 64 MiB reserve: the round it ran in the yield ends
    with again = 1, it is SCHEDULED again with no progress, and its next round runs it in its turn after the fit."""
    big = _device_table([(500_000, 100, 31)])          # 5e7 rows in one device block
    ref = stream_solo(eng, [(big, None)], "EWMA")[0]
    eng.set_fit_sharing(64 * MB)
    job = eng.submit(long_arima[0], algo="ARIMA", tad_id="long", emit_all=True)
    try:
        _wait_fitting(job)
        q = eng.submit_stream(algo="EWMA", tad_id="too-big", share=True)
        q.push(big)
        again = q.end()
        st_q, p_q, state = q.poll(), q.progress(), job.poll()["state"]
        rounds = [again]
        fd = threading.Thread(target=lambda: rounds.extend([feed(q, [(big, None)])]))
        fd.start()
        job.wait()
        t_arima = time.time()
        fd.join()
        st = q.wait()
        t_q = time.time()
        rows_q = q.result()
        q.release()
        assert job.yields()["yields"] >= 1
    finally:
        eng.set_fit_sharing(0)
        job.release()
    print("too large for the reserve: again %d, then %s; ran %.2f s after the fit" % (again, rounds[1:], t_q - t_arima))
    assert again
    assert state == "RUNNING"
    assert st_q["state"] == "SCHEDULED" and st_q["completed_stages"] == 0
    assert p_q == {"passes_done": 0, "passes": 0, "fits_done": 0, "fits_total": 0}
    assert st["state"] == "COMPLETED"
    assert_same_rows(rows_q, ref, what="streamed EWMA too large for the reserve")


def test_cancel_parked_streamed_arima(eng, long_stream, small_stream):
    blocks, _ = long_stream
    small, ref_e = small_stream
    eng.set_memory_budget(ARIMA_BUDGET)
    eng.set_fit_sharing(RESERVE)
    job = eng.submit_stream(algo="ARIMA", tad_id="long", share=True, rows_hint=LONG_SERIES * 100 + LONG_POINTS)
    fd = Feeder(job, blocks)
    fd.start()
    try:
        _wait_fitting(job)
        q = eng.submit_stream(algo="EWMA", tad_id="in-its-place", share=True)
        q.push(small[0][0], text=small[0][1])
        t0 = time.time()
        while q.poll()["state"] != "RUNNING":
            assert time.time() - t0 < 5.0, q.poll()
            time.sleep(0.001)
        job.cancel()
        time.sleep(0.2)
        st_mid = job.poll()["state"]
        for b, txt in small[1:]:
            q.push(b, text=txt)
        assert not q.end()
        st_q = q.wait()
        t_q = time.time()
        st = job.wait(check=False)
        t_a = time.time()
        fd.join()
        rows_q, names_q = q.result(), names_of(q)
        q.release()
    finally:
        job.cancel()                    # a failed check must not leave the feeder waiting
        fd.join()
        eng.set_fit_sharing(0)
        eng.set_memory_budget(0)
        job.release()
    assert st_mid == "RUNNING"                  # the cancel waits for the job running in the fit's place
    assert st["state"] == "FAILED" and st["error"] == TAD_ERR_CANCELLED, st
    assert st_q["state"] == "COMPLETED" and t_a >= t_q - 0.005
    assert fd.error is not None and fd.error.code == TAD_ERR_CANCELLED, fd.error
    assert_same_rows(rows_q, ref_e[0], what="streamed EWMA in a cancelled fit's place")
    same_names(names_q, ref_e[3], "streamed EWMA in a cancelled fit's place")
    # the context runs the next job
    after = stream_solo(eng, small, "EWMA")
    assert_same_rows(after[0], ref_e[0], what="streamed EWMA after the cancel")
