"""Cancel of a multi-GPU job on loopback ranks (W rank contexts on one GPU, test_gpu_loopback_ranks.Ranks): a cancel on
any one rank fails the job on every rank, and no rank is left waiting in a collective.  An ARIMA fit stops within one
evaluation round on every rank through the stop board the ranks map, also while the cancelling rank itself is not
fitting; EWMA and DBSCAN jobs end all FAILED CANCELLED or all COMPLETED, and the next job is exact; a stop for one job
never stops the jobs queued around it.

The loopback runs the ranks' device work in turn, so the times printed here are of ranks that share one GPU."""
import functools
import time

import numpy as np
import pytest

from theia_b200 import sharding, synth
from tests.test_gpu_loopback_ranks import Ranks, check_union, completed, shards_of
from tests.util import assert_same_rows, oracle_rows

pytestmark = pytest.mark.gpu

ERR_CANCELLED = -6
LONG_POINTS = 4_000              # one connection of this many points: its fits alone take minutes
# cancel -> every rank FAILED; the long connection alone needs minutes.  Measured on an H100 80GB HBM3 (700 W) with
# loopback ranks: 0.02 s at W = 2 and 4, under 0.01 s inside passes.
BOUND_S = 15.0


@pytest.fixture
def ranks(monkeypatch):
    made = []

    def make(world, **env):
        rk = Ranks(world, monkeypatch, **env)
        made.append(rk)
        return rk
    yield make
    for rk in made:
        rk.close()


def _noisy(series, points, seed):
    import torch
    t = synth.torch_cols_to_numpy(synth.make_flows_torch(series, points, seed=seed, device=torch.device("cuda", 0),
                                                         noisy=True))
    torch.cuda.synchronize()
    return t


@functools.lru_cache(maxsize=None)
def long_table(world, series, points):
    """`series` noisy connections of `points` points and one of LONG_POINTS whose key rank 0 owns."""
    base = _noisy(series, points, seed=31)
    long = _noisy(1, LONG_POINTS, seed=32)
    for port in range(1024, 65536):
        long["src_port"][:] = port
        if sharding.owner_rank({k: v[:1] for k, v in long.items()}, world, 1 << 20)[0] == 0:
            break
    t = {k: np.concatenate([base[k], long[k]]) for k in base}
    assert (sharding.owner_rank(t, world)[-LONG_POINTS:] == 0).all()
    return t


def _wait(job, cond, what, timeout=300.0):
    t0 = time.time()
    while not cond(job.progress()):
        assert job.poll()["state"] in ("SCHEDULED", "RUNNING"), (what, job.poll())
        assert time.time() - t0 < timeout, what
        time.sleep(0.005)


def _all_cancelled(sts, what):
    for r, st in enumerate(sts):
        assert (st["state"], st["error"]) == ("FAILED", ERR_CANCELLED), (what, r, st["error"], st["err_msg"])
        assert "cancelled" in st["err_msg"], (what, r, st["err_msg"])


def _cancel_mid_fit(rk, table, fitting, budgets=None):
    """Submits `table` as ARIMA on every rank, cancels on rank W-1 once `fitting(progress of rank 0)` holds; returns
    (seconds from the cancel to the last rank FAILED, statuses, rank 0's progress)."""
    W = rk.world
    for e in rk.engs:
        e.set_memory_budget(budgets or 0)
    jobs, cols = rk.submit_all(shards_of(table, W), algo="ARIMA", tad_id="mr-cancel")
    try:
        _wait(jobs[0], fitting, "rank 0's fit")
        t0 = time.time()
        jobs[W - 1].cancel()
        sts = [j.wait(check=False) for j in jobs]
        dt = time.time() - t0
        p = jobs[0].progress()
    finally:
        for j in jobs:
            j.release()
        for c in cols:
            c.free()
        for e in rk.engs:
            e.set_memory_budget(0)
    return dt, sts, p


@pytest.mark.parametrize("world", [2, 4])
def test_cancel_mid_fit(ranks, world):
    """Rank 0 fits a ~4,000-point connection; rank W-1, not fitting (it waits for the device turn or for its peers),
    cancels: rank 0's fit stops within a round and every rank fails CANCELLED; the ranks go on with an exact job."""
    rk = ranks(world)
    t = long_table(world, 100 * world, 100)
    dt, sts, p = _cancel_mid_fit(rk, t, lambda p: p["fits_done"] > 0)
    print("%d ranks: cancel on rank %d -> every rank FAILED in %.3f s, rank 0 at %d of %d fits (H100, loopback)"
          % (world, world - 1, dt, p["fits_done"], p["fits_total"]))
    _all_cancelled(sts, "mid-fit")
    assert p["fits_done"] < p["fits_total"]
    assert dt < BOUND_S
    small = synth.make_flows(500 * world, 40, seed=33)
    sts, got = rk.run(shards_of(small, world), algo="EWMA", tad_id="mr-after", emit_all=True)
    completed(sts, "after a cancel")
    check_union(got, small, "EWMA", "%d ranks after a multi-GPU cancel" % world, emit_all=True)


@pytest.mark.parametrize("world", [2, 4])
def test_cancel_mid_fit_in_passes(ranks, world):
    """The same inside a hash-range pass: the cancel lands while rank 0 fits the pass holding the long connection."""
    from tests.multi_passes_worker import BUDGET_4
    rk = ranks(world)
    t = long_table(world, 20000 * world, 40)
    dt, sts, p = _cancel_mid_fit(rk, t, lambda p: p["fits_done"] > 0 and p["fits_total"] - p["fits_done"] > LONG_POINTS // 2,
                                 budgets=BUDGET_4)
    print("%d ranks in passes: cancel -> every rank FAILED in %.3f s, rank 0 at %d of %d fits, pass %d of %d"
          % (world, dt, p["fits_done"], p["fits_total"], p["passes_done"], p["passes"]))
    _all_cancelled(sts, "mid-fit in passes")
    assert p["passes"] >= 2 and p["fits_done"] < p["fits_total"]
    assert dt < BOUND_S


@pytest.mark.parametrize("env", [{}, {"TAD_OPTIMISTIC": 0}, {"TAD_PEER_PULL": 0}], ids=["default", "exact", "nccl"])
@pytest.mark.parametrize("algo", ["EWMA", "DBSCAN"])
@pytest.mark.parametrize("world", [2, 4])
def test_cancel_agrees(ranks, world, algo, env):
    """A cancel on one rank right after submit, and once its job shows RUNNING: all ranks FAILED CANCELLED or all
    COMPLETED with the oracle's union, never a mix and never an NCCL error; the next job's union is the oracle's."""
    rk = ranks(world, **env)
    table = synth.make_flows(2000 * world, 40, seed=34)
    want, _, _ = oracle_rows(table, algo, emit_all=True)
    for when in ("submit", "running"):
        for cancel_rank in (0, world - 1):
            jobs, cols = rk.submit_all(shards_of(table, world), algo=algo, tad_id="mr-agree", emit_all=True)
            try:
                if when == "running":
                    t0 = time.time()
                    while jobs[cancel_rank].poll()["state"] == "SCHEDULED" and time.time() - t0 < 60:
                        time.sleep(0.0005)
                jobs[cancel_rank].cancel()
                sts = [j.wait(check=False) for j in jobs]
                what = "%s cancel on rank %d at %s" % (algo, cancel_rank, when)
                states = {st["state"] for st in sts}
                assert len(states) == 1, (what, [(s["state"], s["error"], s["err_msg"]) for s in sts])
                if states == {"FAILED"}:
                    _all_cancelled(sts, what)
                else:
                    parts = [j.result() for j in jobs]
                    got = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
                    assert_same_rows(got, want, score_rtol=0, what=what)
            finally:
                for j in jobs:
                    j.release()
                for c in cols:
                    c.free()
            sts, got = rk.run(shards_of(table, world), algo=algo, tad_id="mr-next", emit_all=True)
            completed(sts, "next job")
            assert_same_rows(got, want, score_rtol=0, what="%s next job after a cancel" % algo)


@pytest.mark.parametrize("world", [2, 4])
def test_ordinals(ranks, world):
    """Three ARIMA jobs queued on every rank; the second is cancelled on one rank while the first runs: the first and
    third complete with the union of an uncancelled run on every rank, the second fails on every rank."""
    rk = ranks(world)
    table = _noisy(300 * world, 40, seed=35)
    sts, want = rk.run(shards_of(table, world), algo="ARIMA", tad_id="mr-ref", emit_all=True)
    completed(sts, "reference")
    shards = shards_of(table, world)
    cols = [[e.columns_from_numpy(s) for e, s in zip(rk.engs, shards)] for _ in range(3)]
    jobs = [[e.submit(c[r], algo="ARIMA", tad_id="mr-ord%d" % i, emit_all=True) for r, e in enumerate(rk.engs)]
            for i, c in enumerate(cols)]
    try:
        jobs[1][world - 1].cancel()
        sts = [[j.wait(check=False) for j in js] for js in jobs]
        for i in (0, 2):
            completed(sts[i], "job %d" % i)
            parts = [j.result() for j in jobs[i]]
            got = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
            assert_same_rows(got, want, score_rtol=0, what="job %d around a cancelled one" % i)
        _all_cancelled(sts[1], "the cancelled job")
    finally:
        for js in jobs:
            for j in js:
                j.release()
        for c in cols:
            for x in c:
                x.free()


@pytest.mark.parametrize("world", [2, 4])
def test_release_mid_fit(ranks, world):
    """release() of a fitting ARIMA job on one rank fails it on every rank within the cancel's bound."""
    rk = ranks(world)
    t = long_table(world, 100 * world, 100)
    jobs, cols = rk.submit_all(shards_of(t, world), algo="ARIMA", tad_id="mr-release")
    try:
        _wait(jobs[0], lambda p: p["fits_done"] > 0, "rank 0's fit")
        t0 = time.time()
        jobs[world - 1].release()
        sts = [j.wait(check=False) for j in jobs[:-1]]
        dt = time.time() - t0
        p = jobs[0].progress()
        print("%d ranks: release on rank %d -> the other ranks FAILED in %.3f s, rank 0 at %d of %d fits"
              % (world, world - 1, dt, p["fits_done"], p["fits_total"]))
        _all_cancelled(sts, "release")
        assert p["fits_done"] < p["fits_total"]
        assert dt < BOUND_S
    finally:
        for j in jobs[:-1]:
            j.release()
        for c in cols:
            c.free()
