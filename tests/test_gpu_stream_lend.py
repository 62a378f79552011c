"""Lending (TAD_FLAG_LEND): a streamed job whose caller pauses runs the queued EWMA and DBSCAN tad_submit jobs in the
fit-sharing reserve meanwhile, its own round parked.  Every job's rows, a text job's names, an ARIMA job's fit counts and
the pass counts equal those of a solo run of the same job on the same engine."""
import threading
import time

import pytest

from theia_b200 import synth
from tests.util import assert_same_rows

from .test_gpu_fit_sharing_stream import _host_table, names_of, same_names, text_blocks
from .test_gpu_ns_text import LISTS, _cuts, _namespaces
from .test_gpu_ns_text import blocks as ns_blocks

pytestmark = pytest.mark.gpu

TAD_ERR_CANCELLED = -6
MB = 1 << 20
RESERVE = 256 * MB
BUDGET = 1024 * MB
PASS_BUDGET = RESERVE + 64 * MB     # the streamed job plans in 64 MiB: 2e6 rows run in hash-range passes
HOST = 1 << 30
PAUSE = 0.5                         # the caller's pause, in which the queued jobs must complete


@pytest.fixture(scope="module")
def eng():
    """A context of its own: the budgets and the reserve set here must not reach the session's engine."""
    from theia_b200.engine import TadEngine
    e = TadEngine(device=0)
    yield e
    e.close()


def plain_blocks(table, block):
    n = len(table["flow_end"])
    return [({k: v[lo:lo + block] for k, v in table.items()}, None) for lo in range(0, n, block)]


def push_all(job, blocks):
    for b, txt in blocks:
        job.push(b, text=txt or None)


def feed_rounds(job, blocks, pause=None):
    """Every round until the input is complete; pause(k) is called after round k's end() asked for another round."""
    rounds, again = 0, True
    while again:
        push_all(job, blocks)
        again = job.end()
        rounds += 1
        if again and pause is not None:
            pause(rounds)
    return rounds


def stream_solo(eng, blocks, budget=0, host=0, **kw):
    """The streamed job alone, lending off: (rows, status, names, memory, progress, rounds)."""
    eng.set_fit_sharing(0)
    eng.set_memory_budget(budget)
    eng.set_host_budget(host)
    job = eng.submit_stream(tad_id="solo", **kw)
    try:
        rounds = feed_rounds(job, blocks)
        st = job.wait()
        names = names_of(job) if blocks[0][1] and "src_ip" in blocks[0][1] else None
        return job.result(), st, names, job.memory(), job.progress(), rounds
    finally:
        job.release()
        eng.set_memory_budget(0)
        eng.set_host_budget(0)


class Queued:
    """A tad_submit job's host table, its solo rows and, once submitted, its handle."""

    def __init__(self, eng, table, algo):
        self.eng, self.algo = eng, algo
        self.cols = eng.columns_from_numpy(table)
        job = eng.submit(self.cols, algo=algo, tad_id="solo")
        try:
            job.wait()
            self.ref = job.result()
        finally:
            job.release()
        self.job = None

    def submit(self):
        self.job = self.eng.submit(self.cols, algo=self.algo, tad_id="queued")
        return self

    def state(self):
        return self.job.poll()["state"]

    def check(self, what):
        st = self.job.wait()
        assert_same_rows(self.job.result(), self.ref, what=what)
        return st

    def done(self):
        if self.job is not None:
            self.job.release()
            self.job = None


@pytest.fixture(scope="module")
def small(eng):
    """A 2e5-row table in host blocks, and an EWMA and a DBSCAN table to queue, each with its solo rows."""
    blocks = plain_blocks(synth.make_flows(2_000, 100, seed=61), 8_192)
    q = [Queued(eng, synth.make_flows(500, 100, seed=62), "EWMA"), Queued(eng, synth.make_flows(300, 60, seed=63), "DBSCAN")]
    yield blocks, stream_solo(eng, blocks, budget=BUDGET - RESERVE), q
    for x in q:
        x.cols.free()


@pytest.fixture(scope="module")
def large(eng):
    """Two 4e6-row tables to queue: each runs long enough in the reserve to be seen running."""
    q = [Queued(eng, synth.make_flows(40_000, 100, seed=64 + k), "EWMA") for k in range(2)]
    yield q
    for x in q:
        x.cols.free()


def check_stream(job, ref, what):
    rows, st_ref, names, mem_ref, p_ref, _ = ref
    st = job.wait()
    assert_same_rows(job.result(), rows, what=what)
    if names is not None:
        same_names(names_of(job), names, what)
    mem = job.memory()
    assert mem["passes"] == mem_ref["passes"], what
    assert mem["stored_rows"] == mem_ref["stored_rows"], what
    p = job.progress()
    assert (p["fits_done"], p["fits_total"]) == (p_ref["fits_done"], p_ref["fits_total"]), what
    for k in ("rows_in", "rows_kept", "points", "series", "result_rows"):
        assert st[k] == st_ref[k], (what, k)
    return st, mem, job.lent()


def pause_with(queued, job, timeout=PAUSE):
    """The caller pauses: the queued jobs are submitted and must complete within `timeout` while `job` is RUNNING."""
    for q in queued:
        q.submit()
    t0 = time.time()
    for q in queued:
        q.job.wait(timeout_ms=max(1, int((timeout - (time.time() - t0)) * 1000)), check=False)
    states = [q.state() for q in queued]
    assert states == ["COMPLETED"] * len(queued), states
    assert job.poll()["state"] == "RUNNING"
    return time.time() - t0


def wait_state(q, state, timeout=30.0):
    t0 = time.time()
    while q.state() != state:
        assert time.time() - t0 < timeout, q.job.poll()
        time.sleep(0.001)


def test_mid_round_lend(eng, small):
    blocks, ref, q = small
    eng.set_memory_budget(BUDGET)
    eng.set_fit_sharing(RESERVE)
    job = eng.submit_stream(algo="EWMA", tad_id="lend", lend=True)
    try:
        half = len(blocks) // 2
        push_all(job, blocks[:half])
        dt = pause_with(q, job)
        push_all(job, blocks[half:])
        assert not job.end()
        st, mem, lent = check_stream(job, ref, "streamed EWMA that lent")
        for x in q:
            x.check("%s run in a lend" % x.algo)
            assert x.job.memory()["peak_workspace_bytes"] <= RESERVE
    finally:
        job.cancel()
        job.release()
        for x in q:
            x.done()
        eng.set_fit_sharing(0)
        eng.set_memory_budget(0)
    print("mid-round lend: queued jobs done in %.1f ms; lent %d jobs, %.1f ms; h2d %.1f ms, device %.1f ms"
          % (dt * 1e3, lent["jobs_run"], lent["lent_ms"], st["phase_ms"]["h2d"], st["device_ms"]))
    assert lent["jobs_run"] == 2 and lent["lent_ms"] > 0
    assert mem["peak_workspace_bytes"] <= BUDGET - RESERVE


def test_lend_before_the_first_block_and_between_rounds(eng, small):
    _, _, q = small
    blocks = plain_blocks(synth.make_flows(20_000, 100, seed=65), 65_536)
    n = 20_000 * 100
    ref = stream_solo(eng, blocks, budget=PASS_BUDGET - RESERVE, rows_hint=n, algo="EWMA")
    assert ref[3]["passes"] >= 2 and ref[5] >= 2
    eng.set_memory_budget(PASS_BUDGET)
    eng.set_fit_sharing(RESERVE)
    job = eng.submit_stream(algo="EWMA", tad_id="lend", lend=True, rows_hint=n)
    try:
        pause_with(q[:1], job, timeout=5.0)                 # the context started the job: it waits for its first block
        rounds = feed_rounds(job, blocks, pause=lambda k: pause_with(q[1:], job) if k == 1 else None)
        st, mem, lent = check_stream(job, ref, "streamed EWMA in passes that lent")
        for x in q:
            x.check("%s run in a lend" % x.algo)
    finally:
        job.cancel()
        job.release()
        for x in q:
            x.done()
        eng.set_fit_sharing(0)
        eng.set_memory_budget(0)
    assert rounds == ref[5]
    assert lent["jobs_run"] == 2 and lent["lent_ms"] > 0
    assert mem["peak_workspace_bytes"] <= PASS_BUDGET - RESERVE


def test_device_text_lends_while_its_dictionaries_grow(eng, small):
    _, _, q = small
    t = synth.make_flows(2_000, 100, seed=66)
    n = len(t["flow_end"])
    blocks = ns_blocks(t, _namespaces(n, 3), _cuts(n, 8_192), True, True)
    kw = dict(algo="EWMA", emit_all=True, ns_ignore_names=LISTS[2])
    ref = stream_solo(eng, blocks, budget=BUDGET - RESERVE, **kw)
    eng.set_memory_budget(BUDGET)
    eng.set_fit_sharing(RESERVE)
    job = eng.submit_stream(tad_id="lend", lend=True, **kw)
    try:
        half = len(blocks) // 2
        push_all(job, blocks[:half])
        pause_with(q, job)
        push_all(job, blocks[half:])
        assert not job.end()
        st, mem, lent = check_stream(job, ref, "streamed text job that lent")
        for x in q:
            x.check("%s run in a text job's lend" % x.algo)
    finally:
        job.cancel()
        job.release()
        for x in q:
            x.done()
        eng.set_fit_sharing(0)
        eng.set_memory_budget(0)
    assert st["rows_kept"] < st["rows_in"]
    assert lent["jobs_run"] == 2


def test_push_during_a_lend_waits_for_one_job(eng, small, large):
    blocks, ref, _ = small
    eng.set_memory_budget(BUDGET)
    eng.set_fit_sharing(RESERVE)
    job = eng.submit_stream(algo="EWMA", tad_id="lend", lend=True)
    try:
        half = len(blocks) // 2
        push_all(job, blocks[:half])
        for x in large:
            x.submit()
        wait_state(large[0], "RUNNING")
        t0 = time.time()
        push_all(job, blocks[half:half + 2])      # the first push returns at once, the second once the block is taken
        dt = time.time() - t0
        states = [x.state() for x in large]
        push_all(job, blocks[half + 2:])
        assert not job.end()
        check_stream(job, ref, "streamed EWMA pushed to during a lend")
        for x in large:
            x.check("large EWMA queued beside a lend")
    finally:
        job.cancel()
        job.release()
        for x in large:
            x.done()
        eng.set_fit_sharing(0)
        eng.set_memory_budget(0)
    print("push during a lend returned after %.1f ms" % (dt * 1e3))
    assert states == ["COMPLETED", "SCHEDULED"], states


@pytest.mark.parametrize("lend,reserve", [(False, RESERVE), (True, 0)])
def test_no_flag_or_sharing_off_keeps_the_order(eng, small, lend, reserve):
    blocks, ref, q = small
    eng.set_memory_budget(BUDGET if reserve else BUDGET - RESERVE)
    eng.set_fit_sharing(reserve)
    job = eng.submit_stream(algo="EWMA", tad_id="nolend", lend=lend)
    try:
        half = len(blocks) // 2
        push_all(job, blocks[:half])
        q[0].submit()
        time.sleep(PAUSE / 2)
        state = q[0].state()
        push_all(job, blocks[half:])
        assert not job.end()
        _, _, lent = check_stream(job, ref, "streamed EWMA without lending")
        q[0].check("EWMA behind a streamed job")
    finally:
        job.cancel()
        job.release()
        q[0].done()
        eng.set_fit_sharing(0)
        eng.set_memory_budget(0)
    assert state == "SCHEDULED"
    assert lent == {"jobs_run": 0, "lent_ms": 0.0}


def test_queued_job_too_large_for_the_reserve_waits_its_turn(eng, small):
    blocks, ref, _ = small
    reserve = 64 * MB
    big = Queued(eng, synth.make_flows(1, 600_000, seed=67), "EWMA")     # one connection: 1/64 does not fit 64 MiB
    eng.set_memory_budget(BUDGET - RESERVE + reserve)
    eng.set_fit_sharing(reserve)
    job = eng.submit_stream(algo="EWMA", tad_id="lend", lend=True)
    try:
        half = len(blocks) // 2
        push_all(job, blocks[:half])
        big.submit()
        time.sleep(PAUSE)
        state = big.state()
        push_all(job, blocks[half:])
        assert not job.end()
        _, _, lent = check_stream(job, ref, "streamed EWMA beside a job too large for the reserve")
        big.check("EWMA too large for the reserve")
    finally:
        job.cancel()
        job.release()
        big.done()
        big.cols.free()
        eng.set_fit_sharing(0)
        eng.set_memory_budget(0)
    assert state == "SCHEDULED"
    assert lent["jobs_run"] == 0


def test_cancel_during_a_lend(eng, small, large):
    blocks, _, q = small
    eng.set_memory_budget(BUDGET)
    eng.set_fit_sharing(RESERVE)
    job = eng.submit_stream(algo="EWMA", tad_id="lend", lend=True)
    errors = []

    def feeder():
        try:
            push_all(job, blocks[half:half + 2])
        except Exception as e:          # checked below
            errors.append(e)

    try:
        half = len(blocks) // 2
        push_all(job, blocks[:half])
        large[0].submit()
        wait_state(large[0], "RUNNING")
        fd = threading.Thread(target=feeder)
        fd.start()
        time.sleep(0.002)
        job.cancel()
        fd.join()
        st = job.wait(check=False)
        large[0].check("EWMA lent to a job cancelled meanwhile")
        # the context runs the next job correctly
        q[0].submit()
        q[0].check("EWMA after a cancelled lend")
    finally:
        job.cancel()
        job.release()
        large[0].done()
        q[0].done()
        eng.set_fit_sharing(0)
        eng.set_memory_budget(0)
    assert st["state"] == "FAILED" and st["error"] == TAD_ERR_CANCELLED
    assert len(errors) == 1 and getattr(errors[0], "code", None) == TAD_ERR_CANCELLED, errors


def test_memory_with_a_host_store_round(eng, small):
    """The lending job's first round goes to the host row store: the out-stage and the partly filled staging are parked
    through the lend.  Its peak stays in the budget less the reserve, the lent jobs' in the reserve."""
    _, _, q = small
    blocks = plain_blocks(synth.make_flows(20_000, 100, seed=68), 65_536)
    n = 20_000 * 100
    ref = stream_solo(eng, blocks, budget=PASS_BUDGET - RESERVE, host=HOST, rows_hint=n, algo="EWMA")
    assert ref[3]["passes"] >= 2 and ref[3]["stored_rows"] > 0 and ref[5] == 1
    eng.set_memory_budget(PASS_BUDGET)
    eng.set_host_budget(HOST)
    eng.set_fit_sharing(RESERVE)
    job = eng.submit_stream(algo="EWMA", tad_id="lend", lend=True, rows_hint=n)
    try:
        half = len(blocks) // 2 + 1
        push_all(job, blocks[:half])
        pause_with(q, job)
        push_all(job, blocks[half:])
        assert not job.end()
        _, mem, lent = check_stream(job, ref, "streamed EWMA to the host store that lent")
        peaks = [x.job.memory()["peak_workspace_bytes"] for x in q]
        for x in q:
            x.check("%s run in a store round's lend" % x.algo)
    finally:
        job.cancel()
        job.release()
        for x in q:
            x.done()
        eng.set_fit_sharing(0)
        eng.set_host_budget(0)
        eng.set_memory_budget(0)
    assert lent["jobs_run"] == 2
    assert mem["peak_workspace_bytes"] <= PASS_BUDGET - RESERVE
    assert all(p <= RESERVE for p in peaks), peaks
    assert mem["peak_host_bytes"] <= HOST


def test_streamed_arima_lends_and_yields(eng, small):
    _, _, q = small
    # the 2,000-point connection gives a fit phase of a few seconds: the queued job finds it running
    t = _host_table([(30_000, 100, 69), (1, 2_000, 70)])
    blocks = plain_blocks(t, 65_536)
    ref = stream_solo(eng, blocks, budget=BUDGET - RESERVE, algo="ARIMA", emit_all=True)
    eng.set_memory_budget(BUDGET)
    eng.set_fit_sharing(RESERVE)
    job = eng.submit_stream(algo="ARIMA", tad_id="lend", emit_all=True, share=True, lend=True)
    try:
        half = len(blocks) // 2
        push_all(job, blocks[:half])
        pause_with(q[:1], job)
        # a one-pass job's last tad_stream_end returns once its result is published: the rest is fed from a thread
        errors = []

        def rest():
            try:
                push_all(job, blocks[half:])
                assert not job.end()
            except Exception as e:      # checked below
                errors.append(e)

        fd = threading.Thread(target=rest)
        fd.start()
        t0 = time.time()
        while job.progress()["fits_done"] == 0:
            assert time.time() - t0 < 120, job.poll()
            time.sleep(0.002)
        time.sleep(0.2)
        q[1].submit()
        q[1].job.wait()
        fit_state = job.poll()["state"]
        fd.join()
        assert not errors, errors
        _, _, lent = check_stream(job, ref, "streamed ARIMA that lent and yielded")
        y = job.yields()
        for x in q:
            x.check("%s beside a streamed ARIMA job" % x.algo)
    finally:
        job.cancel()
        job.release()
        for x in q:
            x.done()
        eng.set_fit_sharing(0)
        eng.set_memory_budget(0)
    print("streamed ARIMA: lent %d jobs (%.1f ms), %d yields (%.1f ms parked)"
          % (lent["jobs_run"], lent["lent_ms"], y["yields"], y["parked_ms"]))
    assert fit_state == "RUNNING"
    assert lent["jobs_run"] >= 1 and lent["lent_ms"] > 0
    assert y["yields"] >= 1 and y["parked_ms"] > 0
