"""The multi-rank paths on ONE GPU: W rank engines on device 0, joined by a loopback id (TadEngine.loopback_id) instead of
NCCL, run every partition and exchange path that otherwise needs W GPUs.  The union of the ranks' rows must equal the C
oracle bit for bit (ARIMA: the single-GPU engine's one-shot run), every rank must own exactly the rows the host mirror
of the key hash gives it, and the histogram phase must run exactly when the optimistic partition was not taken.

Covered here and nowhere else on a one-GPU machine: segment descriptors with nseg > 1 (seg_span over counts or offsets),
the fused EWMA instance's segment walk, the spill gather across segments, the segment scan with the pull skip, the peer
counter gather, 8 ranks x 4 exchange chunks (32 segments, kMaxSeg), the hash-range passes of a rank job and their agreed
split, cancel and NOMEM verdicts.  The loopback serialises the ranks' device work, so no timing here means anything;
the real IPC mappings, NVLink reads and NCCL are covered only by the torchrun tests (test_multi_rank*.py)."""
import functools
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from theia_b200 import sharding, synth
from tests import adversarial as A
from tests.util import assert_same_rows, oracle_rows

pytestmark = pytest.mark.gpu

MB = 1 << 20
ERR_NOMEM, ERR_CANCELLED, ERR_UNSUPPORTED = -3, -6, -7
SWITCHES = ("TAD_PEER_PULL", "TAD_EXACT_PULL", "TAD_EXCHANGE_CHUNKS", "TAD_EXCHANGE_MIN_ROWS", "TAD_DEBUG_LOGB",
            "TAD_OPTIMISTIC")


class Ranks:
    """``world`` rank engines on device 0 in this process, created under one set of run-time switches (every rank must
    see the same values; tad_init reads them)."""

    def __init__(self, world, monkeypatch, **env):
        from theia_b200.engine import TadEngine
        for k in SWITCHES:
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, str(v))
        uid = TadEngine.loopback_id(world)
        self.world = world
        self.engs = []
        try:
            for r in range(world):
                self.engs.append(TadEngine(device=0, world_size=world, rank=r, nccl_unique_id=uid))
        except Exception:
            self.close()
            raise
        finally:
            TadEngine.release_loopback_id(uid)      # no other context joins these ranks
        for k in env:
            monkeypatch.delenv(k)

    def submit_all(self, shards, device=False, **kw):
        """Submits shard r on rank r, from pinned host columns or (``device``) device-resident ones; returns (jobs,
        columns)."""
        if device:
            import torch
            from tests.multi_passes_worker import device_cols
            cols = [device_cols(s) for s in shards]
            torch.cuda.synchronize()                 # the engines' streams do not wait for torch's
        else:
            cols = [e.columns_from_numpy(s) for e, s in zip(self.engs, shards)]
        jobs = []
        for e, c in zip(self.engs, cols):
            jobs.append(e.submit(c, **kw))
        return jobs, cols

    def run(self, shards, budgets=None, cancel_rank=None, device=False, **kw):
        """Every rank's job on its shard: ([status], union of the result rows or None when a rank failed)."""
        for r, e in enumerate(self.engs):
            if budgets is not None:
                e.set_memory_budget(budgets[r] if isinstance(budgets, (list, tuple)) else budgets)
        jobs, cols = self.submit_all(shards, device, **kw)
        if cancel_rank is not None:
            jobs[cancel_rank].cancel()
        try:
            # the workers run on their own: waiting on one rank after another blocks no rank
            sts = [j.wait(check=False) for j in jobs]
            for j, st in zip(jobs, sts):
                if st["state"] == "COMPLETED":
                    st.update(j.memory())
                    st["progress"] = j.progress()
            parts = [j.result() for j in jobs] if all(s["state"] == "COMPLETED" for s in sts) else None
        finally:
            for j in jobs:
                j.release()
            for c in cols:
                c.free()
        union = None if parts is None else {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
        return sts, union

    def close(self):
        # tad_shutdown meets the peers (their exported buffers outlive every mapping): close every rank at once
        with ThreadPoolExecutor(max(1, len(self.engs))) as ex:
            list(ex.map(lambda e: e.close(), self.engs))
        self.engs = []


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


def shards_of(table, world):
    return [sharding.shard_rows(table, r, world) for r in range(world)]


def completed(sts, what):
    for r, st in enumerate(sts):
        assert st["state"] == "COMPLETED", (what, r, st["error"], st["err_msg"])


def check_owned(sts, table, world, what, start_time=0, end_time=0):
    """Rows owned after the time window (flow_start >= start, flow_end < end; 0 = unbounded) per the host mirror."""
    own = sharding.owner_rank(table, world, len(table["flow_end"]))
    keep = np.ones(len(own), dtype=bool)
    if start_time:
        keep &= table["flow_start"] >= start_time
    if end_time:
        keep &= table["flow_end"] < end_time
    assert [st["rows_owned"] for st in sts] == [int(((own == r) & keep).sum()) for r in range(world)], what


def check_union(got, table, algo, what, **kw):
    want, ns, npts = oracle_rows(table, algo, **kw)
    assert_same_rows(got, want, score_rtol=0, what=what)


# ---------------------------------------------------------------------------------------------------------------------
# Paths x world sizes
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def flows(name, scale=1):
    """multi_worker.py's tables, the second one (scale 2) larger: a spread table (long connections shuffled over the
    ranks), and a skewed one (two 6000-point connections: a slot overflows, every rank takes the exact partition)."""
    table = synth.make_flows(4000 * scale, 40, seed=77 + scale, dup_frac=0.05, ragged=True)
    if name == "skewed":
        t2 = synth.make_flows(2, 6000, seed=78)
        return {k: np.concatenate([table[k], t2[k]]) for k in table}
    t2 = synth.make_flows(3, 900, seed=79)
    table = {k: np.concatenate([table[k], t2[k]]) for k in table}
    perm = np.random.default_rng(5 + scale).permutation(len(table["value"]))
    return {k: v[perm] for k, v in table.items()}


# path -> (table, switches, optimistic partition taken)
PATHS = {
    "pull": ("spread", {}, True),
    "exact_pull": ("skewed", {}, False),
    "exact_nccl": ("skewed", {"TAD_EXACT_PULL": 0}, False),
    "nccl_k1": ("spread", {"TAD_PEER_PULL": 0, "TAD_EXCHANGE_MIN_ROWS": 0, "TAD_EXCHANGE_CHUNKS": 1}, False),
    "nccl_k2": ("spread", {"TAD_PEER_PULL": 0, "TAD_EXCHANGE_MIN_ROWS": 0, "TAD_EXCHANGE_CHUNKS": 2}, False),
    "nccl_k4": ("spread", {"TAD_PEER_PULL": 0, "TAD_EXCHANGE_MIN_ROWS": 0, "TAD_EXCHANGE_CHUNKS": 4}, False),
}


@functools.lru_cache(maxsize=None)
def arima_table():
    import torch
    t = synth.torch_cols_to_numpy(synth.make_flows_torch(1500, 40, seed=88, device=torch.device("cuda", 0), noisy=True))
    torch.cuda.synchronize()
    return t


@functools.lru_cache(maxsize=None)
def arima_one_gpu(emit_all):
    """The single-GPU engine's one-shot ARIMA run (no rank engine is running meanwhile)."""
    from theia_b200.engine import TadEngine
    with TadEngine(device=0) as eng:
        got, _ = eng.run(arima_table(), algo="ARIMA", tad_id="loopback-ref", emit_all=emit_all)
    return got


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("world", [2, 4, 8])
def test_paths(ranks, world, path):
    """Each path at each world size, one engine set for two tables in a row (the second larger: the exported buffer is
    reused, then regrown), EWMA and DBSCAN with emit_all on and off and both reducers, and ARIMA."""
    name, env, optimistic = PATHS[path]
    arima_want = {e: arima_one_gpu(e) for e in (False, True)}
    rk = ranks(world, **env)
    runs = ((1, "EWMA", True, 0), (1, "DBSCAN", False, 1), (2, "EWMA", False, 1), (2, "DBSCAN", True, 0),
            (1, "EWMA", True, 1))
    for scale, algo, emit_all, reducer in runs:
        table = flows(name, scale)
        total = len(table["value"])
        what = "%d ranks, %s, x%d, %s emit_all=%s reducer=%d" % (world, path, scale, algo, emit_all, reducer)
        # global_rows: given by the host on the first table, agreed on by the ranks on the second
        sts, got = rk.run(shards_of(table, world), algo=algo, tad_id="loopback", emit_all=emit_all, reducer=reducer,
                          global_rows=total if scale == 1 else 0)
        completed(sts, what)
        check_owned(sts, table, world, what)
        assert [st["rows_kept"] for st in sts] == [len(s["value"]) for s in shards_of(table, world)], what
        assert [st["phase_ms"]["hist"] == 0.0 for st in sts] == [optimistic] * world, (what, [s["phase_ms"] for s in sts])
        check_union(got, table, algo, what, emit_all=emit_all, reducer=reducer)
    for emit_all in (False, True):
        t = arima_table()
        sts, got = rk.run(shards_of(t, world), algo="ARIMA", tad_id="loopback", emit_all=emit_all)
        completed(sts, "ARIMA")
        check_owned(sts, t, world, "ARIMA")
        assert_same_rows(got, arima_want[emit_all], score_rtol=0,
                         what="%d ranks, %s, ARIMA emit_all=%s vs one GPU" % (world, path, emit_all))


# ---------------------------------------------------------------------------------------------------------------------
# Adversarial tables
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def adv(name):
    return {
        "collision": lambda: A.collision_table(seed=11),
        "one_bucket": lambda: A.one_bucket_table(seed=15),
        "lattice": lambda: A.dbscan_lattice_table(seed=17),
        "ewma": lambda: A.ewma_edge_table(seed=18),
        "timestamps": lambda: A.timestamp_table(seed=19),
        "duplicates": lambda: A.duplicate_table(seed=20),
    }[name]()


def adv_check(rk, table, algo, what, **kw):
    sts, got = rk.run(shards_of(table, rk.world), algo=algo, tad_id="loopback-adv", **kw)
    completed(sts, what)
    check_owned(sts, table, rk.world, what, kw.get("start_time", 0), kw.get("end_time", 0))
    want, ns, npts = oracle_rows(table, algo, **kw)
    assert sum(st["series"] for st in sts) == ns and sum(st["points"] for st in sts) == npts, what
    assert_same_rows(got, want, score_rtol=0, what="%s %s %s" % (what, algo, kw))
    return sts


@pytest.mark.parametrize("exchange", ["pull", "nccl"])
@pytest.mark.parametrize("world", [2, 8])
def test_adversarial(ranks, world, exchange):
    """Every generator of tests/adversarial.py on the rank engines: colliding keys and protocol twins (one owner each),
    the overfull bucket (every rank falls back to the exact partition; its spill gathers the bucket from W segments),
    eps lattices, strict EWMA flags, timestamps and wrapping duplicate sums."""
    env = {} if exchange == "pull" else {"TAD_PEER_PULL": 0, "TAD_EXCHANGE_MIN_ROWS": 0, "TAD_EXCHANGE_CHUNKS": 2}
    rk = ranks(world, **env)
    what = "%d ranks %s" % (world, exchange)
    t, info = adv("collision")
    for algo in ("EWMA", "DBSCAN"):
        for emit_all in (False, True):
            sts = adv_check(rk, t, algo, what + " collision", emit_all=emit_all)
            assert sum(st["series"] for st in sts) == info["series"]
    t, info = adv("one_bucket")
    for algo in ("EWMA", "DBSCAN"):
        sts = adv_check(rk, t, algo, what + " one bucket")
        assert sum(st["spill_rows"] for st in sts) == info["rows"]
        assert all(st["phase_ms"]["hist"] > 0 for st in sts)
    t, _ = adv("lattice")
    for emit_all in (False, True):
        adv_check(rk, t, "DBSCAN", what + " lattice", emit_all=emit_all)
    adv_check(rk, t, "EWMA", what + " lattice", emit_all=True)
    t, _ = adv("ewma")
    for algo in ("EWMA", "DBSCAN"):
        adv_check(rk, t, algo, what + " ewma edges", emit_all=True)
    adv_check(rk, t, "EWMA", what + " ewma edges")
    t, info = adv("timestamps")
    for reducer in (0, 1):
        for algo in ("EWMA", "DBSCAN"):
            adv_check(rk, t, algo, what + " timestamps", reducer=reducer, emit_all=True)
        adv_check(rk, t, "EWMA", what + " timestamps window", reducer=reducer, emit_all=True,
                  start_time=info["start_time"], end_time=info["end_time"])
    t, _ = adv("duplicates")
    for reducer in (0, 1):
        for algo in ("EWMA", "DBSCAN"):
            adv_check(rk, t, algo, what + " duplicates", reducer=reducer, emit_all=reducer == 1)


@pytest.mark.parametrize("world", [2, 8])
def test_probe_chains(ranks, world):
    """A bucket of exactly a class's capacity whose probes all wrap (16 buckets), at every class, pulled from W
    sources."""
    rk = ranks(world, TAD_DEBUG_LOGB=4)
    for cap in A.CLASS_CAPS:
        t, _ = A.probe_chain_table(cap, 3, seed=21)
        for algo, emit_all in (("EWMA", True), ("DBSCAN", True), ("EWMA", False)):
            adv_check(rk, t, algo, "%d ranks probe %d" % (world, cap), emit_all=emit_all)


# ---------------------------------------------------------------------------------------------------------------------
# Capacity classes assembled from several segments
# ---------------------------------------------------------------------------------------------------------------------
LOGB = 4
# rows of bucket b (16 buckets): both sides of the 512-, 768- and 1280-row capacities, every class's capacity, kGroupCap
# (4096) itself, a small and a one-row bucket, and an empty one
SIZES = [511, 512, 513, 767, 768, 769, 1024, 1279, 1280, 1281, 1536, 2048, 4096, 100, 1, 0]


def class_shards(points, world, seed):
    """Shards in which bucket b's rows come from one source (b % 3 == 0, where that fits a source's slot), from every
    source (b % 3 == 1, and the b % 3 == 0 buckets too large for one slot) or from every source but one (b % 3 == 2: a
    source with none of its rows), dealt out evenly, so that no slot of the optimistic partition overflows."""
    pool = synth.make_flows(140_000 // points, points, seed=seed)
    bucket = sharding.key_hash(pool) >> np.uint64(64 - LOGB)
    slot = max(256, 4096 // world)          # tad_engine.cu: slot()
    rng = np.random.default_rng(seed)
    per_src = [[] for _ in range(world)]
    for b, n in enumerate(SIZES):
        rows = np.flatnonzero(bucket == b)[:n]
        assert len(rows) == n
        if b % 3 == 0 and n <= slot:
            srcs = [b % world]
        elif b % 3 == 2:
            srcs = [s for s in range(world) if s != b % world]
        else:
            srcs = list(range(world))
        src = np.asarray(srcs)[(np.arange(n) + b) % len(srcs)]
        for s in range(world):
            per_src[s].append(rows[src == s])
    idx = [rng.permutation(np.concatenate(p)) for p in per_src]
    shards = [{k: v[i] for k, v in pool.items()} for i in idx]
    table = {k: np.concatenate([s[k] for s in shards]) for k in pool}
    return shards, table


@pytest.mark.parametrize("exchange", ["pull", "nccl"])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_classes_from_segments(ranks, world, exchange):
    """Every capacity class filled from W sources (TAD_DEBUG_LOGB=4): buckets held by one source, by all, by all but
    one, and one of kGroupCap rows; one point per connection (every class's hash table at its highest load) and 20."""
    env = {"TAD_DEBUG_LOGB": LOGB}
    if exchange == "nccl":
        env.update(TAD_PEER_PULL=0, TAD_EXCHANGE_MIN_ROWS=0, TAD_EXCHANGE_CHUNKS=4)
    rk = ranks(world, **env)
    for points in (1, 20):
        shards, table = class_shards(points, world, seed=90 + points)
        for algo, kw in (("EWMA", {"emit_all": True}), ("DBSCAN", {"emit_all": True}), ("EWMA", {"reducer": 1})):
            what = "%d ranks %s classes, %d points, %s %s" % (world, exchange, points, algo, kw)
            sts, got = rk.run(shards, algo=algo, tad_id="loopback-classes", **kw)
            completed(sts, what)
            check_owned(sts, table, world, what)
            assert sum(st["spill_rows"] for st in sts) == 0, what
            assert [st["phase_ms"]["hist"] == 0.0 for st in sts] == [exchange == "pull"] * world, what
            check_union(got, table, algo, what, **kw)


# ---------------------------------------------------------------------------------------------------------------------
# Hash-range passes (the scenarios of tests/multi_passes_worker.py)
# ---------------------------------------------------------------------------------------------------------------------
def _passes_agree(sts, what, budgets):
    completed(sts, what)
    assert len({st["passes"] for st in sts}) == 1, (what, [st["passes"] for st in sts])
    for r, st in enumerate(sts):
        assert st["peak_workspace_bytes"] <= budgets[r], (what, r, st["peak_workspace_bytes"], budgets[r])
        assert st["progress"]["passes_done"] == st["progress"]["passes"] == st["passes"], (what, r, st["progress"])
    return sts[0]["passes"]


@pytest.mark.parametrize("world", [2, 4])
def test_passes(ranks, world):
    """P >= 2 and P >= 4 equal the oracle; skewed ownership; unequal budgets agree on one P; a cancel on one rank and a
    1/64 range that does not fit fail every rank alike, and the contexts run the next job."""
    from tests.multi_passes_worker import BUDGET_2, BUDGET_4, ROOMY, case_table
    rk = ranks(world)
    W = world
    spread = case_table("spread", W)
    for algo in ("EWMA", "DBSCAN"):
        for budget, at_least in ((0, 1), (BUDGET_2, 2), (BUDGET_4, 4)):
            what = "%d ranks spread %s budget %d MiB" % (W, algo, budget >> 20)
            sts, got = rk.run(shards_of(spread, W), budgets=budget, algo=algo, tad_id="lp-passes", emit_all=True)
            p = _passes_agree(sts, what, [budget or 1 << 62] * W)
            assert p >= at_least, (what, p)
            check_owned(sts, spread, W, what)
            check_union(got, spread, algo, what, emit_all=True)
    # device-resident input: each pass is one split launch over the rank's device columns
    for algo in ("EWMA", "DBSCAN"):
        for budget, at_least in ((0, 1), (BUDGET_4, 4)):
            what = "%d ranks spread %s device input budget %d MiB" % (W, algo, budget >> 20)
            sts, got = rk.run(shards_of(spread, W), budgets=budget, device=True, algo=algo, tad_id="lp-passes",
                              emit_all=True)
            assert _passes_agree(sts, what, [budget or 1 << 62] * W) >= at_least, what
            check_owned(sts, spread, W, what)
            check_union(got, spread, algo, what, emit_all=True)
    skewed = case_table("skewed", W)
    sts, got = rk.run(shards_of(skewed, W), budgets=BUDGET_4, algo="EWMA", tad_id="lp-passes", emit_all=True)
    _passes_agree(sts, "skewed", [BUDGET_4] * W)
    owned = [st["rows_owned"] for st in sts]
    assert owned[-1] > 2 * max(owned[:-1]), owned
    check_owned(sts, skewed, W, "skewed")
    check_union(got, skewed, "EWMA", "%d ranks skewed 64 MiB" % W, emit_all=True)
    unequal = [BUDGET_4] + [ROOMY] * (W - 1)
    sts, got = rk.run(shards_of(spread, W), budgets=unequal, algo="EWMA", tad_id="lp-passes", emit_all=True)
    planned = _passes_agree(sts, "unequal", unequal)
    assert planned >= 4, planned
    check_union(got, spread, "EWMA", "%d ranks unequal budgets" % W, emit_all=True)
    # ARIMA in passes equals its one-pass run on the same ranks
    t = synth.torch_cols_to_numpy(synth.make_flows_torch(20000 * W, 40, seed=88, device=__import__("torch").device("cuda", 0),
                                                         noisy=True))
    __import__("torch").cuda.synchronize()
    sts, one = rk.run(shards_of(t, W), budgets=0, algo="ARIMA", tad_id="lp-passes", emit_all=True)
    completed(sts, "ARIMA one pass")
    sts, got = rk.run(shards_of(t, W), budgets=BUDGET_4, algo="ARIMA", tad_id="lp-passes", emit_all=True)
    assert _passes_agree(sts, "ARIMA", [BUDGET_4] * W) >= 2
    assert_same_rows(got, one, score_rtol=0, what="%d ranks ARIMA in passes vs one pass" % W)
    # a cancel on rank 0 right after submit: every rank fails CANCELLED; then the contexts go on
    sts, _ = rk.run(shards_of(spread, W), budgets=BUDGET_4, cancel_rank=0, algo="EWMA", tad_id="lp-cancel", emit_all=True)
    assert [(st["state"], st["error"]) for st in sts] == [("FAILED", ERR_CANCELLED)] * W, [st["err_msg"] for st in sts]
    assert all("cancelled" in st["err_msg"] for st in sts)
    small = case_table("small", W)
    sts, got = rk.run(shards_of(small, W), budgets=BUDGET_4, algo="EWMA", tad_id="lp-passes", emit_all=True)
    _passes_agree(sts, "after cancel", [BUDGET_4] * W)
    check_union(got, small, "EWMA", "%d ranks after a cancel" % W, emit_all=True)
    # a 1/64 range that does not fit: every rank fails NOMEM, naming the rank and the bytes; then the contexts go on
    sts, _ = rk.run(shards_of(case_table("one_big", W), W), budgets=BUDGET_4, algo="EWMA", tad_id="lp-nomem",
                    emit_all=True)
    assert [(st["state"], st["error"]) for st in sts] == [("FAILED", ERR_NOMEM)] * W, [st["err_msg"] for st in sts]
    assert all("rank" in st["err_msg"] and "bytes" in st["err_msg"] for st in sts), [st["err_msg"] for st in sts]
    sts, got = rk.run(shards_of(small, W), budgets=BUDGET_4, algo="DBSCAN", tad_id="lp-passes", emit_all=True)
    _passes_agree(sts, "after NOMEM", [BUDGET_4] * W)
    check_union(got, small, "DBSCAN", "%d ranks after NOMEM" % W, emit_all=True)


@pytest.mark.parametrize("world", [2, 4])
def test_passes_split_and_exchange(ranks, world):
    """One bucket per rank (TAD_DEBUG_LOGB): rank 0's passes do not fit its budget, every rank splits them together;
    and the chunked NCCL exchange inside the passes."""
    from tests.multi_passes_worker import BUDGET_4, ROOMY, case_table
    W = world
    spread = case_table("spread", W)
    unequal = [BUDGET_4] + [ROOMY] * (W - 1)
    rk = ranks(W)
    sts, _ = rk.run(shards_of(spread, W), budgets=unequal, algo="EWMA", tad_id="lp-split", emit_all=True)
    planned = _passes_agree(sts, "unequal", unequal)
    rk.close()
    rk = ranks(W, TAD_DEBUG_LOGB=(W - 1).bit_length())
    sts, got = rk.run(shards_of(spread, W), budgets=unequal, algo="EWMA", tad_id="lp-split", emit_all=True)
    split = _passes_agree(sts, "split", unequal)
    assert split > planned, (split, planned)
    assert all(st["spill_rows"] > 0 for st in sts)
    check_union(got, spread, "EWMA", "%d ranks agreed split" % W, emit_all=True)
    rk.close()
    # the NCCL exchange inside the passes, in 4 chunks and in 1: every pass's largest shard is above the chunking
    # threshold, so each pass of the chunked run launches its histogram, scan and scatter once per chunk
    min_rows = len(sharding.shard_rows(spread, 0, W)["value"]) // 64
    per_pass = {}
    for k in (4, 1):
        rk = ranks(W, TAD_PEER_PULL=0, TAD_EXCHANGE_MIN_ROWS=min_rows, TAD_EXCHANGE_CHUNKS=k)
        what = "%d ranks exchange in %d chunks in passes" % (W, k)
        sts, got = rk.run(shards_of(spread, W), budgets=BUDGET_4, algo="EWMA", tad_id="lp-nccl", emit_all=True)
        assert _passes_agree(sts, what, [BUDGET_4] * W) >= 4
        assert all(st["phase_ms"]["hist"] > 0 for st in sts), (what, [st["phase_ms"] for st in sts])
        check_union(got, spread, "EWMA", what, emit_all=True)
        per_pass[k] = [st["gpu_launches"] / st["passes"] for st in sts]
        rk.close()
    # 3 x (4 - 1) more launches per pass when every chunk holds rows; at least two of the three kernels per extra chunk
    assert all(c4 >= c1 + 6 for c4, c1 in zip(per_pass[4], per_pass[1])), per_pass


# ---------------------------------------------------------------------------------------------------------------------
# Refusals
# ---------------------------------------------------------------------------------------------------------------------
def test_rank_engine_refusals(ranks):
    """A rank engine refuses streamed jobs and fit sharing (TAD_ERR_UNSUPPORTED), and runs a job afterwards."""
    from theia_b200.engine import TadError
    rk = ranks(2)
    for e in rk.engs:
        job = e.submit_stream(algo="EWMA", check=False)
        try:
            st = job.poll()
            assert (st["state"], st["error"]) == ("FAILED", ERR_UNSUPPORTED), st
        finally:
            job.release()
        with pytest.raises(TadError) as ei:
            e.set_fit_sharing(64 * MB)
        assert ei.value.code == ERR_UNSUPPORTED
    table = flows("spread")
    sts, got = rk.run(shards_of(table, 2), algo="EWMA", tad_id="lp-refusals", emit_all=True)
    completed(sts, "after the refusals")
    check_union(got, table, "EWMA", "2 ranks after the refusals", emit_all=True)
