"""The adversarial tables of tests/adversarial.py through every partition path, bit for bit against the C oracle:
distinct keys with one 64-bit hash and protocol twins that are neighbours in the spill sort, probe chains that wrap
in every capacity class, a bucket that overfills the optimistic scatter's overflow list, DBSCAN lattices with eps ties
at magnitudes up to 2^64, EWMA series whose flags hinge on the strict compare, timestamps over the whole u32 range,
thousands of duplicates of one point, and pass residues skewed onto one value.

Engines: the default one (optimistic partition), the exact partition (TAD_OPTIMISTIC=0), two buckets (TAD_DEBUG_LOGB=1:
every table of more than about 8k rows spills whole) and 16 buckets (TAD_DEBUG_LOGB=4: probe chains at every class)."""
import functools
import json
import os

import numpy as np
import pytest

from tests import adversarial as A
from tests.test_gpu_group_detect import make_engine
from tests.util import assert_same_rows, oracle_rows

pytestmark = pytest.mark.gpu

MB = 1 << 20
BUDGET_FLOOR = 64 * MB
ERR_NOMEM = -3
ENV = {"exact": {"TAD_OPTIMISTIC": "0"}, "logb1": {"TAD_DEBUG_LOGB": "1"}, "logb4": {"TAD_DEBUG_LOGB": "4"}}
COUNTS = ("rows_in", "rows_kept", "points", "series", "result_rows")


@pytest.fixture(scope="module")
def engines(engine):
    e = {name: make_engine(**env) for name, env in ENV.items()}
    e["default"] = engine
    yield e
    for name in ENV:
        e[name].close()


@functools.lru_cache(maxsize=None)
def table(name):
    return {
        "collision": lambda: A.collision_table(seed=11),
        "collision_big": lambda: A.collision_table(seed=12, filler_series=55_000, filler_points=20),
        "arima": A.arima_collision_table,
        "arima_big": lambda: A.collision_table(seed=14, groups=40, filler_series=130_000, filler_points=8, twin_points=30,
                                               noisy=True),
        "one_bucket": lambda: A.one_bucket_table(seed=15),
        "skewed": lambda: A.skewed_residue_table(seed=16),
        "lattice": lambda: A.dbscan_lattice_table(seed=17),
        "ewma": lambda: A.ewma_edge_table(seed=18),
        "timestamps": lambda: A.timestamp_table(seed=19),
        "duplicates": lambda: A.duplicate_table(seed=20),
    }[name]()


@functools.lru_cache(maxsize=None)
def _oracle(name, algo, kw):
    return oracle_rows(table(name)[0], algo, **dict(kw))


def want(name, algo, **kw):
    return _oracle(name, algo, tuple(sorted(kw.items())))


def check(eng, name, algo, what="", **kw):
    t, info = table(name)
    got, st = eng.run(t, algo=algo, tad_id="adversarial", **kw)
    w, ns, npts = want(name, algo, **kw)
    assert st["state"] == "COMPLETED"
    assert st["series"] == ns and st["points"] == npts, (name, algo, kw, st["series"], ns, st["points"], npts)
    assert st["result_rows"] == len(w["flow_end"])
    assert_same_rows(got, w, what="%s %s %s %s" % (what, name, algo, kw))
    return got, st


ALL = ["default", "exact", "logb1", "logb4"]


@pytest.mark.parametrize("emit_all", [False, True])
@pytest.mark.parametrize("algo", ["EWMA", "DBSCAN"])
@pytest.mark.parametrize("which", ALL)
def test_collisions(engines, which, algo, emit_all):
    """Distinct keys with one 64-bit hash share bucket, tag and start slot: only the group kernel's full-key compare
    and the spill sort's key columns keep their series apart.  The protocol twins' rows are neighbours in the spill
    sort, where only the key head's protocol compare splits them."""
    _, st = check(engines[which], "collision", algo, which, emit_all=emit_all)
    assert st["series"] == table("collision")[1]["series"]
    assert st["spill_rows"] >= 2 * 2100


_probe_tables = {}


@pytest.mark.parametrize("points", [1, 3])
@pytest.mark.parametrize("cap", A.CLASS_CAPS)
def test_probe_chains(engines, cap, points):
    """A bucket of exactly `cap` rows whose probes all start at slot HT-1: the linear probe wraps to 0 and the chain
    covers two thirds of the table; a fifth of the keys share the whole tag.  The bucket fits its class: nothing
    spills."""
    name = "probe_%d_%d" % (cap, points)
    if name not in _probe_tables:
        _probe_tables[name] = A.probe_chain_table(cap, points, seed=21)
    t, info = _probe_tables[name]
    for algo, emit_all in (("EWMA", True), ("DBSCAN", True), ("EWMA", False)):
        got, st = engines["logb4"].run(t, algo=algo, tad_id="probe", emit_all=emit_all)
        w, ns, npts = oracle_rows(t, algo, emit_all=emit_all)
        assert st["spill_rows"] == 0
        assert st["series"] == ns and st["points"] == npts, (st["series"], ns)
        assert_same_rows(got, w, what="%s %s" % (name, algo))
    got, st = engines["default"].run(t, algo="EWMA", emit_all=True)
    assert_same_rows(got, oracle_rows(t, "EWMA", emit_all=True)[0], what=name + " default")


@pytest.mark.parametrize("algo", ["EWMA", "DBSCAN"])
def test_one_bucket_forces_the_exact_fallback(engines, algo):
    """1.2M rows in one bucket overfill the overflow list: the partition falls back to the exact one (the histogram
    phase runs only there; device-resident input, so the phase is timed on its own) and the spill path takes the whole
    bucket of 300k series."""
    from tests.test_gpu_passes import _device_cols
    t, info = table("one_bucket")
    eng = engines["default"]
    import torch
    cols = _device_cols(t)
    torch.cuda.synchronize()                   # the engine's stream does not wait for torch's
    job = eng.submit(cols, algo=algo, tad_id="one-bucket")
    try:
        st = job.wait()
        got = job.result()
    finally:
        job.release()
        cols.free()
    w, ns, npts = want("one_bucket", algo)
    assert st["series"] == ns == info["series"] and st["points"] == npts
    assert_same_rows(got, w, what="one bucket " + algo)
    assert st["phase_ms"]["hist"] > 0
    assert st["spill_rows"] == info["rows"]


@pytest.mark.parametrize("emit_all", [False, True])
@pytest.mark.parametrize("which", ALL)
def test_dbscan_lattice(engines, which, emit_all):
    """Eps ties, border points and chains at magnitudes up to 2^64, series of 4 to 6000 points: the brute-force rule
    (n <= 11), the two-pointer sweep with the group kernel's value ranks (up to 4096 points) and the spill path's own
    ranking (4097 and 6000 points; on the two-bucket engine every series)."""
    check(engines[which], "lattice", "DBSCAN", which, emit_all=emit_all)
    if emit_all:
        check(engines[which], "lattice", "EWMA", which, emit_all=True)


@pytest.mark.parametrize("emit_all", [False, True])
@pytest.mark.parametrize("which", ALL)
def test_ewma_edges(engines, which, emit_all):
    """Constant, all-zero and 0 / 2^64-1 series and values at 2^53 -+ 1, 2^63 and 2^64-1, of 1, 2, 4095, 4096 and 4097
    points: the flag compare is strict, the reciprocal table's last entry and the spill path's division agree."""
    _, st = check(engines[which], "ewma", "EWMA", which, emit_all=emit_all)
    if which == "default":
        assert st["spill_rows"] == 6 * 4097          # every 4097-point series, and only those
    check(engines[which], "ewma", "DBSCAN", which, emit_all=emit_all)


@pytest.mark.parametrize("reducer", [0, 1])
@pytest.mark.parametrize("which", ALL)
def test_timestamps(engines, which, reducer):
    """Times over [0, 2^32-1], bursts inside one bin, rows in descending order; filters whose bounds equal row times."""
    info = table("timestamps")[1]
    for algo in ("EWMA", "DBSCAN"):
        check(engines[which], "timestamps", algo, which, reducer=reducer, emit_all=True)
    check(engines[which], "timestamps", "EWMA", which, reducer=reducer, emit_all=True, start_time=info["start_time"],
          end_time=info["end_time"])


@pytest.mark.parametrize("emit_all", [False, True])
@pytest.mark.parametrize("reducer", [0, 1])
@pytest.mark.parametrize("which", ALL)
def test_duplicates(engines, which, reducer, emit_all):
    """4096 copies of one point (one time bin, one value after the reduce), 16 x 256 copies, 4097 copies on the spill
    path; values near 2^62, so the sum reducer wraps past 2^64."""
    for algo in ("EWMA", "DBSCAN"):
        check(engines[which], "duplicates", algo, which, reducer=reducer, emit_all=emit_all)


# --------------------------------------------------------------------------------------------------------------------
# ARIMA: scores are not pinned against the oracle; the series, keys, times, throughputs and stddevs are
# --------------------------------------------------------------------------------------------------------------------
GOLDEN_ARIMA = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "adversarial_arima_series.json")


def _key_rows(cols):
    return np.stack([np.asarray(cols[c]).astype(np.int64) for c in ("src_ip", "src_port", "dst_ip", "dst_port", "proto",
                                                                    "flow_start")], 1)


def test_arima_on_collisions(engines):
    """ARIMA on a small table of collision groups, protocol twins and noisy filler (about 900 series of up to 40
    points): the one-shot, exact-partition and all-spilled runs agree bit for bit; the series they score are those the
    ARIMA oracle keeps (committed by tests/golden/make_adversarial_arima.py) but for two named short-prefix optimiser
    cases, with the oracle's keys, times, throughputs and stddevs."""
    t, info = table("arima")
    golden = json.load(open(GOLDEN_ARIMA))
    assert golden["sha256"] == A.table_digest(t), "the table changed: regenerate " + GOLDEN_ARIMA
    assert golden["key_columns"] == ["src_ip", "src_port", "dst_ip", "dst_port", "proto", "flow_start"]
    got, st = engines["default"].run(t, algo="ARIMA", tad_id="arima", emit_all=True)
    spill, st_s = engines["logb1"].run(t, algo="ARIMA", tad_id="arima", emit_all=True)
    exact, st_x = engines["exact"].run(t, algo="ARIMA", tad_id="arima", emit_all=True)
    assert st_s["spill_rows"] == st_s["rows_kept"]
    for other, so, what in ((spill, st_s, "all spilled"), (exact, st_x, "exact")):
        for k in COUNTS:
            assert so[k] == st[k], (what, k)
        assert_same_rows(other, got, what="ARIMA " + what + " vs one-shot")
    from oracle import tad_oracle as o
    g = o.canonicalize(got)
    kept = {tuple(r) for r in golden["kept"]}
    assert len(kept) >= 100
    scored = {tuple(r) for r in _key_rows(g).tolist()}
    # Two series of 825 differ, both decided by the fit of a 3- or 4-point prefix, where the two L-BFGS implementations
    # end in different local optima (oracle/arima_oracle.py): one whose 3-point forecast the oracle puts at -5331 (a NaN
    # after the inverse Box-Cox at lambda 2.6), one of 4 points at lambda -6.4 (its inverse overflows for forecasts above
    # 0.16).  Any other series scored or dropped against the oracle fails here.
    assert len(scored ^ kept) <= 2, sorted(scored ^ kept)
    both = scored & kept
    g = {c: v[np.array([tuple(r) in both for r in _key_rows(g).tolist()], dtype=bool)] for c, v in g.items()}
    w, _, _ = oracle_rows(t, "EWMA", emit_all=True)
    sel = np.array([tuple(r) in both for r in _key_rows(w).tolist()], dtype=bool)
    w = {c: v[sel] for c, v in w.items()}
    assert len(g["flow_end"]) == len(w["flow_end"])
    for c in ("src_ip", "src_port", "dst_ip", "dst_port", "proto", "flow_start", "flow_end", "throughput", "stddev"):
        assert np.array_equal(g[c], w[c], equal_nan=True), c


# --------------------------------------------------------------------------------------------------------------------
# hash-range passes under a memory budget
# --------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def peng():
    """A context of its own: the budgets set here must not reach the session's engine."""
    from theia_b200.engine import TadEngine
    e = TadEngine(device=0)
    yield e
    e.close()


def run_budget(eng, t, budget, check=True, **kw):
    eng.set_memory_budget(budget)
    cols = eng.columns_from_numpy(t)
    job = eng.submit(cols, tad_id="passes", **kw)
    try:
        st = job.wait(check=check)
        if st["state"] != "COMPLETED":
            return None, st, None
        return job.result(), st, job.memory()
    finally:
        job.release()
        cols.free()


def same_as(got, st, ref, st_ref, what):
    for k in COUNTS:
        assert st[k] == st_ref[k], (what, k, st[k], st_ref[k])
    assert_same_rows(got, ref, what=what)


@pytest.mark.parametrize("algo", ["EWMA", "DBSCAN"])
def test_collisions_in_passes(peng, algo):
    """1.1M rows at the budget floor: two passes or more, each holding whole collision groups and twins (one hash, one
    pass), bit-identical to one pass and to the oracle."""
    t, _ = table("collision_big")
    ref, st_ref, mem_ref = run_budget(peng, t, 0, algo=algo, emit_all=True)
    assert mem_ref["passes"] == 1
    got, st, mem = run_budget(peng, t, BUDGET_FLOOR, algo=algo, emit_all=True)
    assert mem["passes"] >= 2 and mem["peak_workspace_bytes"] <= BUDGET_FLOOR, mem
    same_as(got, st, ref, st_ref, "%s passes vs one pass" % algo)
    w, ns, npts = want("collision_big", algo, emit_all=True)
    assert st["series"] == ns and st["points"] == npts
    assert_same_rows(got, w, what="%s passes vs oracle" % algo)


def test_arima_collisions_across_passes(peng, engines):
    """ARIMA on ~1M rows of collision groups and short noisy series: one pass, two passes or more at the budget floor,
    and every bucket spilled (two-bucket engine) give the same rows bit for bit."""
    t, _ = table("arima_big")
    ref, st_ref, mem_ref = run_budget(peng, t, 0, algo="ARIMA", emit_all=True)
    assert mem_ref["passes"] == 1
    got, st, mem = run_budget(peng, t, BUDGET_FLOOR, algo="ARIMA", emit_all=True)
    assert mem["passes"] >= 2 and mem["peak_workspace_bytes"] <= BUDGET_FLOOR, mem
    same_as(got, st, ref, st_ref, "ARIMA passes vs one pass")
    spill, st_s = engines["logb1"].run(t, algo="ARIMA", tad_id="arima", emit_all=True)
    assert st_s["spill_rows"] == st_s["rows_kept"]
    same_as(spill, st_s, ref, st_ref, "ARIMA all spilled vs one pass")


def test_skewed_residues():
    """80 % of the rows (1.6M of 2M) share the low 6 hash bits, so halving the passes never splits the heavy residue.

    With emit_all the planner knows every pass's result size, so the pass count comes from the plan alone.  The budgets
    are derived from the one-pass workspace W of this table (an exact-partition pass of all rows).  At 0.9 W the whole
    table does not fit and neither does the 90 % that the first of two passes holds, but the heavy residue does: the
    plan has to come from the residue counts and takes at least four passes (a plan from uniform residues would take
    two and overfill the first).  Without emit_all nearly every point of these short series is flagged, so a pass's
    result outgrows its first-guess buffer while it runs; at 0.75 W the heavy residue's result rows do not fit, the job
    fails with TAD_ERR_NOMEM naming the result buffer, and at the budget floor the plan itself fails.  The context then
    runs a normal job correctly."""
    from theia_b200.engine import TadEngine
    t, info = table("skewed")
    with TadEngine(device=0) as e:
        ref, st_ref, mem_ref = run_budget(e, t, 300 * MB, emit_all=True)      # one exact-partition pass
        assert mem_ref["passes"] == 1
        w = mem_ref["peak_workspace_bytes"]
        want_rows, _, _ = want("skewed", "EWMA", emit_all=True)
        assert_same_rows(ref, want_rows, what="skewed vs oracle")
        budget = int(0.9 * w)
        got, st, mem = run_budget(e, t, budget, emit_all=True)
        assert 4 <= mem["passes"] <= 64 and mem["peak_workspace_bytes"] <= budget, (budget, mem)
        same_as(got, st, ref, st_ref, "skewed in passes, budget %d" % budget)
        _, st, _ = run_budget(e, t, int(0.75 * w), check=False)
        assert st["state"] == "FAILED" and st["error"] == ERR_NOMEM, st
        assert "result buffer" in st["err_msg"] and "budget" in st["err_msg"], st["err_msg"]
        _, st, _ = run_budget(e, t, BUDGET_FLOOR, check=False)
        assert st["state"] == "FAILED" and st["error"] == ERR_NOMEM, st
        assert "budget" in st["err_msg"], st["err_msg"]
        got, st, _ = run_budget(e, table("collision")[0], BUDGET_FLOOR, emit_all=True)
        assert_same_rows(got, want("collision", "EWMA", emit_all=True)[0], what="after a failed job")


# --------------------------------------------------------------------------------------------------------------------
# streamed input
# --------------------------------------------------------------------------------------------------------------------
def block_source(t):
    """Every round in its own row order, cut into blocks of 1 to 65536 rows."""
    n = len(t["flow_end"])
    rounds = [0]

    def factory():
        rng = np.random.default_rng(500 + rounds[0])
        rounds[0] += 1
        perm = rng.permutation(n)
        cuts = [0]
        while cuts[-1] < n:
            cuts.append(min(n, cuts[-1] + int(rng.choice([1, 7, 2047, 4096, 30000, 65536]))))
        for lo, hi in zip(cuts[:-1], cuts[1:]):
            yield {c: np.ascontiguousarray(v[perm[lo:hi]]) for c, v in t.items()}
    return factory


@pytest.mark.parametrize("reducer", [0, 1])
@pytest.mark.parametrize("algo", ["EWMA", "DBSCAN"])
@pytest.mark.parametrize("name", ["collision", "timestamps", "duplicates"])
def test_streamed(engines, name, algo, reducer):
    eng = engines["default"]
    t, _ = table(name)
    ref, st_ref = eng.run(t, algo=algo, reducer=reducer, emit_all=True, tad_id="one-shot")
    got, st = eng.run_stream(block_source(t), algo=algo, reducer=reducer, emit_all=True, tad_id="stream")
    assert st["state"] == "COMPLETED"
    same_as(got, st, ref, st_ref, "streamed %s %s reducer %d" % (name, algo, reducer))
    w, ns, npts = want(name, algo, reducer=reducer, emit_all=True)
    assert st["series"] == ns and st["points"] == npts
    assert_same_rows(got, w, what="streamed vs oracle")
