"""Jobs streamed to every rank (TAD_FLAG_RANK_STREAM) on ONE GPU: W rank engines on device 0 joined by a loopback id, as
in test_gpu_loopback_ranks.py, each fed from a thread of its own.  The rows are dealt to the ranks at random, not by
owner, and each rank's share is cut into uneven host and device blocks.  The union of the ranks' rows must equal the C
oracle bit for bit (ARIMA: the same ranks' one-shot tad_submit run); the ranks must agree on the pass count and on
every round's *again; and every verdict must fail every rank alike and leave the contexts able to run the next job.

The loopback serialises the ranks' device work and maps no memory over IPC, so no timing here means anything, and the
NVLink reads and NCCL calls are covered only by test_gpu_multi_rank_stream.py."""
import threading

import numpy as np
import pytest

from theia_b200 import synth
from tests.test_gpu_loopback_ranks import Ranks, flows, shards_of
from tests.util import assert_same_rows, oracle_rows

pytestmark = pytest.mark.gpu

MB = 1 << 20
ERR_INVALID_ARG, ERR_NOMEM, ERR_CANCELLED, ERR_UNSUPPORTED = -1, -3, -6, -7
FEEDER_WAIT_S = 120


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


def deal(table, world, seed, empty_rank=None):
    """Every row to a random rank (not its owner); `empty_rank` gets none."""
    n = len(table["flow_end"])
    to = np.random.default_rng(seed).integers(0, world, n)
    if empty_rank is not None:
        to[to == empty_rank] = (empty_rank + 1) % world
    return [{k: v[to == r] for k, v in table.items()} for r in range(world)]


def cut(share, seed, device):
    """Uneven blocks of one rank's share; with `device`, every other block is device-resident."""
    from tests.test_gpu_stream import device_cols
    n = len(share["flow_end"])
    rng = np.random.default_rng(seed)
    cuts = [0]
    while cuts[-1] < n:
        cuts.append(min(n, cuts[-1] + int(rng.choice([1, 97, 2047, 30000, 65536, 400000]))))
    blocks = []
    for k, (lo, hi) in enumerate(zip(cuts[:-1], cuts[1:])):
        part = {c: v[lo:hi] for c, v in share.items()}
        blocks.append(device_cols(part) if device and k % 2 else part)
    return blocks


class Feeder(threading.Thread):
    """One rank's caller: pushes its blocks round after round while end() asks for them again.  `hook(job, rnd, k)` runs
    before block k of round rnd and returns False to skip the block, or "stop" to return without pushing or ending."""

    def __init__(self, job, blocks, hook=None):
        super().__init__(daemon=True)
        self.job, self.blocks, self.hook = job, blocks, hook
        self.agains, self.code = [], None

    def run(self):
        from theia_b200.engine import TadError
        try:
            rnd = 0
            while True:
                for k, b in enumerate(self.blocks):
                    h = self.hook(self.job, rnd, k) if self.hook else True
                    if h == "stop":
                        return
                    if h:
                        self.job.push(b)
                again = self.job.end()
                self.agains.append(again)
                if not again:
                    return
                rnd += 1
        except TadError as e:
            self.code = e.code


def stream_run(rk, shares, budgets=None, hints=None, device=True, hooks=None, release_rank=None, **kw):
    """Every rank's part of one job streamed to all ranks: ([status], union of the rows or None, [feeder])."""
    W = rk.world
    for r, e in enumerate(rk.engs):
        e.set_memory_budget(budgets[r] if isinstance(budgets, (list, tuple)) else (budgets or 0))
    hints = hints if hints is not None else [len(s["flow_end"]) for s in shares]
    blocks = [cut(s, 31 + r, device) for r, s in enumerate(shares)]
    jobs = [e.submit_stream(ranks=True, rows_hint=hints[r], tad_id="lp-stream", **kw) for r, e in enumerate(rk.engs)]
    feeders = [Feeder(j, b, (hooks or {}).get(r)) for r, (j, b) in enumerate(zip(jobs, blocks))]
    try:
        for f in feeders:
            f.start()
        if release_rank is not None:
            feeders[release_rank].join(FEEDER_WAIT_S)
            jobs[release_rank].release()
        for f in feeders:
            f.join(FEEDER_WAIT_S)
        assert not any(f.is_alive() for f in feeders), "a feeder did not return"
        sts = []
        for r, j in enumerate(jobs):
            if r == release_rank:
                sts.append(None)
                continue
            st = j.wait(check=False)
            if st["state"] == "COMPLETED":
                st.update(j.memory())
            sts.append(st)
        ok = all(st is not None and st["state"] == "COMPLETED" for st in sts)
        parts = [j.result() for j in jobs] if ok else None
    finally:
        for j in jobs:
            j.release()
    union = None if parts is None else {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
    return sts, union, feeders


def completed(sts, feeders, what):
    for r, st in enumerate(sts):
        assert st["state"] == "COMPLETED", (what, r, st["error"], st["err_msg"])
    assert len({st["passes"] for st in sts}) == 1, (what, [st["passes"] for st in sts])
    assert len({tuple(f.agains) for f in feeders}) == 1, (what, [f.agains for f in feeders])
    return sts[0]["passes"], len(feeders[0].agains)


def failed_alike(sts, code, what):
    live = [st for st in sts if st is not None]
    assert [(st["state"], st["error"]) for st in live] == [("FAILED", code)] * len(live), \
        (what, [(st["state"], st["error"], st["err_msg"]) for st in live])
    return [st["err_msg"] for st in live]


def check_oracle(got, table, algo, what, **kw):
    want, _, _ = oracle_rows(table, algo, **kw)
    assert_same_rows(got, want, score_rtol=0, what=what)


def next_job_ok(rk, what):
    table = flows("spread")
    sts, got, fs = stream_run(rk, deal(table, rk.world, 9), budgets=64 * MB, algo="EWMA", emit_all=True)
    completed(sts, fs, what)
    check_oracle(got, table, "EWMA", what, emit_all=True)


@pytest.mark.parametrize("world", [2, 4])
def test_parity_passes_and_rounds(ranks, world):
    """EWMA and DBSCAN equal the oracle in one pass and in passes (BUDGET_2, BUDGET_4, unequal budgets); the ranks agree
    on the pass count and every *again; exact hints cost no extra round, hint 0 at most one; skewed ownership and a rank
    with an empty share work."""
    from tests.multi_passes_worker import BUDGET_2, BUDGET_4, ROOMY, case_table
    rk = ranks(world)
    W = world
    small = flows("spread")
    for algo in ("EWMA", "DBSCAN"):
        sts, got, fs = stream_run(rk, deal(small, W, 1), algo=algo, emit_all=True)
        passes, rounds = completed(sts, fs, "%s one pass" % algo)
        assert (passes, rounds) == (1, 1), (algo, passes, rounds)
        check_oracle(got, small, algo, "%d ranks %s streamed, one pass" % (W, algo), emit_all=True)
    spread = case_table("spread", W)
    for budget, at_least in ((BUDGET_2, 2), (BUDGET_4, 4), ([BUDGET_4] + [ROOMY] * (W - 1), 4)):
        for algo in ("EWMA", "DBSCAN"):
            what = "%d ranks spread %s budget %s" % (W, algo, budget)
            sts, got, fs = stream_run(rk, deal(spread, W, 2), budgets=budget, algo=algo, emit_all=True)
            passes, rounds = completed(sts, fs, what)
            assert passes >= at_least and rounds == passes, (what, passes, rounds)
            for r, st in enumerate(sts):
                b = budget[r] if isinstance(budget, list) else budget
                assert st["peak_workspace_bytes"] <= b, (what, r, st["peak_workspace_bytes"], b)
            check_oracle(got, spread, algo, what, emit_all=True)
    what = "%d ranks hint 0" % W
    sts, got, fs = stream_run(rk, deal(spread, W, 3), budgets=BUDGET_4, hints=[0] * W, algo="EWMA", emit_all=True)
    passes, rounds = completed(sts, fs, what)
    assert passes >= 4 and rounds <= passes + 1, (what, passes, rounds)
    check_oracle(got, spread, "EWMA", what, emit_all=True)
    skewed = case_table("skewed", W)
    what = "%d ranks skewed, rank 0 empty" % W
    sts, got, fs = stream_run(rk, deal(skewed, W, 4, empty_rank=0), budgets=BUDGET_4, algo="EWMA", emit_all=True)
    completed(sts, fs, what)
    owned = [st["rows_owned"] for st in sts]
    assert owned[-1] > 2 * max(owned[:-1]) and sts[0]["rows_in"] == 0, (owned, sts[0]["rows_in"])
    check_oracle(got, skewed, "EWMA", what, emit_all=True)


@pytest.mark.parametrize("world", [2, 4])
def test_wrong_hints_and_count_only(ranks, world):
    """A hint far below or far above the share (a placeholder of 1, 1/20 of it, 30 times it) costs at most one round and
    never a different result or a NOMEM; and a first round whose pass columns may not grow (TAD_DEBUG_NO_GROW) only
    counts, after which the passes are swept into columns again and equal the oracle."""
    from tests.multi_passes_worker import BUDGET_4, ROOMY, case_table
    W = world
    spread = case_table("spread", W)
    shares = deal(spread, W, 14)
    rows = [len(s["flow_end"]) for s in shares]
    rk = ranks(W)
    for budget in (BUDGET_4, ROOMY):
        for name, hints in (("1", [1] * W), ("1/20", [n // 20 for n in rows]), ("30x", [30 * n for n in rows])):
            what = "%d ranks hint %s budget %d MiB" % (W, name, budget >> 20)
            sts, got, fs = stream_run(rk, shares, budgets=budget, hints=hints, algo="EWMA", emit_all=True)
            passes, rounds = completed(sts, fs, what)
            assert rounds <= passes + 1, (what, passes, rounds)
            for r, st in enumerate(sts):
                assert st["peak_workspace_bytes"] <= budget, (what, r, st["peak_workspace_bytes"])
            check_oracle(got, spread, "EWMA", what, emit_all=True)
    rk.close()
    rk = ranks(W, TAD_DEBUG_NO_GROW=1)
    for algo in ("EWMA", "DBSCAN"):
        what = "%d ranks count-only first round %s" % (W, algo)
        sts, got, fs = stream_run(rk, shares, budgets=ROOMY, hints=[0] * W, algo=algo, emit_all=True)
        passes, rounds = completed(sts, fs, what)
        assert rounds == passes + 1, (what, passes, rounds)      # pass 0 was only counted: one round more
        check_oracle(got, spread, algo, what, emit_all=True)


@pytest.mark.parametrize("world", [2, 4])
def test_filters_reducers_and_arima(ranks, world):
    """The time window, u32 namespace ids and the sum reducer equal the oracle; ARIMA equals the same ranks' one-shot
    run of the same table."""
    from tests.multi_passes_worker import BUDGET_4
    rk = ranks(world)
    t = synth.make_flows(2000, 60, seed=82, dup_frac=0.3)
    rng = np.random.default_rng(82)
    n = len(t["value"])
    t["src_ns"] = rng.integers(0, 6, n).astype(np.uint32)
    t["dst_ns"] = rng.integers(0, 6, n).astype(np.uint32)
    win = dict(start_time=synth.T0 + 600, end_time=synth.T0 + 3000, emit_all=True)
    keep = ~np.isin(t["src_ns"], (1, 4)) & ~np.isin(t["dst_ns"], (1, 4))
    plain = {k: v[keep] for k, v in t.items() if k not in ("src_ns", "dst_ns")}
    for reducer in (0, 1):
        for budget in (0, BUDGET_4):
            what = "%d ranks filters reducer %d budget %d" % (world, reducer, budget)
            sts, got, fs = stream_run(rk, deal(t, world, 5), budgets=budget, device=False, reducer=reducer,
                                      ns_ignore=(1, 4), **win)
            completed(sts, fs, what)
            assert sum(st["rows_kept"] for st in sts) < n
            check_oracle(got, plain, "EWMA", what, reducer=reducer, **win)
    import torch
    a = synth.torch_cols_to_numpy(synth.make_flows_torch(1500, 40, seed=88, device=torch.device("cuda", 0), noisy=True))
    torch.cuda.synchronize()
    sts, one = rk.run(shards_of(a, world), budgets=0, algo="ARIMA", tad_id="lp-stream-ref", emit_all=True)
    assert all(st["state"] == "COMPLETED" for st in sts), [st["err_msg"] for st in sts]
    for budget in (0, BUDGET_4):
        sts, got, fs = stream_run(rk, deal(a, world, 6), budgets=budget, algo="ARIMA", emit_all=True)
        completed(sts, fs, "ARIMA budget %d" % budget)
        assert_same_rows(got, one, score_rtol=0, what="%d ranks streamed ARIMA budget %d vs one shot" % (world, budget))


@pytest.mark.parametrize("env", [{"TAD_PEER_PULL": 0}, {"TAD_OPTIMISTIC": 0}], ids=["all_to_all", "exact"])
def test_exchange_paths(ranks, env):
    """The NCCL all-to-all (no peer pull) and the exact partition give the oracle's rows too."""
    from tests.multi_passes_worker import BUDGET_4
    rk = ranks(4, **env)
    table = flows("spread", 2)
    for budget in (0, BUDGET_4):
        for algo in ("EWMA", "DBSCAN"):
            what = "%s budget %d %s" % (env, budget, algo)
            sts, got, fs = stream_run(rk, deal(table, 4, 7), budgets=budget, algo=algo, emit_all=True)
            completed(sts, fs, what)
            check_oracle(got, table, algo, what, emit_all=True)


@pytest.mark.parametrize("world", [2, 4])
def test_verdicts(ranks, world):
    """Each verdict fails every rank alike and the contexts run the next job: a second round that omits a block, a cancel
    on rank 0 mid-round, a release of rank 1 without end, a 1/64 range that fits no budget, and text key columns."""
    from tests.multi_passes_worker import BUDGET_4, case_table
    rk = ranks(world)
    W = world
    spread = case_table("spread", W)

    def last_block(shares):             # rank 1's blocks are cut with seed 32 (stream_run)
        return len(cut(shares[1], 32, False)) - 1

    # rank 1's second round omits its last block: INVALID_ARG naming rank 1
    shares = deal(spread, W, 8)
    last = last_block(shares)
    sts, _, fs = stream_run(rk, shares, budgets=BUDGET_4, algo="EWMA",
                            hooks={1: lambda j, rnd, k: not (rnd == 1 and k == last)})
    msgs = failed_alike(sts, ERR_INVALID_ARG, "omitted block")
    assert all("rank 1" in m for m in msgs), msgs
    next_job_ok(rk, "after an omitted block")

    # a cancel on rank 0 in the middle of its first round: CANCELLED everywhere, the callers' calls return CANCELLED
    def cancel_mid(job, rnd, k):
        if rnd == 0 and k == 2:
            job.cancel()
        return True
    sts, _, fs = stream_run(rk, deal(spread, W, 10), budgets=BUDGET_4, algo="EWMA", hooks={0: cancel_mid})
    msgs = failed_alike(sts, ERR_CANCELLED, "cancel")
    assert all("rank 0" in m for m in msgs), msgs
    assert [f.code for f in fs] == [ERR_CANCELLED] * W, [f.code for f in fs]
    next_job_ok(rk, "after a cancel")

    # rank 1's caller pushes its first round and stops without end; its job is released: every feeder returns
    shares = deal(spread, W, 11)
    last = last_block(shares)
    sts, _, fs = stream_run(rk, shares, budgets=BUDGET_4, algo="EWMA",
                            hooks={1: lambda j, rnd, k: "stop" if k == last else True}, release_rank=1)
    failed_alike(sts, ERR_CANCELLED, "release without end")
    next_job_ok(rk, "after a release")

    # a 1/64 hash range that fits no budget: NOMEM naming the rank and the bytes
    sts, _, fs = stream_run(rk, deal(case_table("one_big", W), W, 12), budgets=BUDGET_4, algo="EWMA")
    msgs = failed_alike(sts, ERR_NOMEM, "nomem")
    assert all("rank" in m and "bytes" in m for m in msgs), msgs
    next_job_ok(rk, "after NOMEM")

    # text key columns on a rank stream job: UNSUPPORTED for the call and for the job on every rank
    def text_push(job, rnd, k):
        from theia_b200.engine import TadError
        if k == 1:
            b = {"flow_end": np.zeros(3, np.uint32), "value": np.zeros(3, np.uint64)}
            with pytest.raises(TadError) as ei:
                job.push(b, text={"src_ip": (b"\x01a\x01b\x01c", np.zeros(1, np.uint64))})
            assert ei.value.code == ERR_UNSUPPORTED
            return "stop"
        return True
    sts, _, fs = stream_run(rk, deal(spread, W, 13), budgets=BUDGET_4, algo="EWMA", hooks={0: text_push})
    failed_alike(sts, ERR_UNSUPPORTED, "push_text")
    next_job_ok(rk, "after push_text")
