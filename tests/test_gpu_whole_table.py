"""Full-size EWMA and DBSCAN jobs checked row for row against the columnar oracle (oracle/columnar_oracle.py), which
tests/test_columnar_oracle.py pins bit for bit to the C oracle.  The sampled checks of test_gpu_full_size.py and
test_gpu_passes_1e9.py see 0.3 % of the series; paths that only run at large bucket counts are checked here on every
row:

* configs[1] (10^8 rows, 10^6 connections x 100 points) on the default engine, with exact series / point / result
  counts: the oracle groups by the full key, as the engine does;
* the same table at 2^18, 2^20 and 2^22 buckets (TAD_DEBUG_LOGB), where every thread of bucket_scan_kernel and
  series_scan_kernel scans 2, 8 and 32 buckets on a 132-SM H100 (the capacity-class lists, the ascending big_list,
  the series hint table over runs of empty buckets), and a 10^5-row table at 2^22 buckets, almost all empty, against
  the C oracle;
* a lumpy 10^8-row table: series of 1 to 6,000 points (thousands of buckets take the spill path, some series past the
  kernels' 4,096-entry reciprocal table), 5 % duplicate rows under both reducers, values within 1e10 of 2^64; the same
  table at 2^18, 2^20 and 2^22 buckets, where the spill rows the engine reports must equal the host's count of rows in
  buckets past 4,096 rows at that bucket count; emit_all on a 10^7-row one; and 10^7-row ones (for DBSCAN with values
  spread far beyond eps) where more points are flagged than the first result-capacity guess holds, so detect runs a
  second time and writes millions of rows;
* 10^9 rows in hash-range passes from pinned host columns.  Its oracle takes minutes, so it runs only when the
  environment sets TAD_TEST_WHOLE_1E9=1; otherwise it skips and says so.

Every case prints its engine and oracle wall times (pytest -s)."""
import os
import resource
import time

import numpy as np
import pytest

from oracle import columnar_oracle as co
from tests.test_gpu_group_detect import make_engine
from tests.util import EXACT_COLS, SCORE_COLS, assert_same_rows, oracle_rows
from theia_b200 import sharding, synth

pytestmark = pytest.mark.gpu

ALGO = {"EWMA": co.ALGO_EWMA, "DBSCAN": co.ALGO_DBSCAN}
GROUP_CAP = 4096                   # rows a bucket may hold to be grouped in shared memory (tad_common.cuh: kGroupCap)
SCAN_MAX_CTAS = 128                # tad_kernels.cu: kScanMaxCtas
U64_MAX = (1 << 64) - 1


def _cuda():
    import torch
    return torch.device("cuda", 0)


def _mem_available():
    try:
        for line in open("/proc/meminfo"):
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    except OSError:
        pass
    return 0


def run_engine(engine, cols, **kw):
    """(rows, status with the job's hash-range ``passes``, engine seconds) of one job on Columns / DeviceColumns."""
    t0 = time.perf_counter()
    job = engine.submit(cols, tad_id="whole", **kw)
    st = job.wait()
    res = job.result()
    st["passes"] = job.memory()["passes"]
    job.release()
    return res, st, time.perf_counter() - t0


def run_oracle(table, algo, **kw):
    t0 = time.perf_counter()
    cols, ns, npts = co.run_job(table, algo=ALGO[algo], sort_device=_cuda(), **kw)
    return (cols, ns, npts), time.perf_counter() - t0


def check_rows(got, st, want, what):
    """Every result row and the series / point / result counts equal the oracle's."""
    cols, ns, npts = want
    assert st["state"] == "COMPLETED", st
    assert (st["series"], st["points"], st["result_rows"]) == (ns, npts, len(cols["flow_end"])), (what, st, ns, npts)
    got = co.canonicalize(got, _cuda())
    assert len(got["flow_end"]) == len(cols["flow_end"]), what
    for c in EXACT_COLS:
        assert np.array_equal(got[c], cols[c]), "%s: column %s differs in %d rows" % (
            what, c, int(np.sum(got[c] != cols[c])))
    for c in SCORE_COLS:
        bad = ~((got[c] == cols[c]) | (np.isnan(got[c]) & np.isnan(cols[c])))
        assert not bad.any(), "%s: %s differs in %d rows, first at %s" % (
            what, c, int(bad.sum()), {k: v[np.flatnonzero(bad)[0]] for k, v in got.items()})


def report(what, engine_s, oracle_s, st, **extra):
    if "passes" in st:
        extra = dict(passes=st["passes"], **extra)
    print("\n[whole table] %s: engine %.1f s (device %.0f ms), oracle %.1f s; series %d, points %d, result rows %d, "
          "spill rows %d%s" % (what, engine_s, st["device_ms"], oracle_s, st["series"], st["points"], st["result_rows"],
                               st["spill_rows"], "".join(", %s %s" % kv for kv in extra.items())))


def scan_per(logb):
    """Buckets each thread of bucket_scan_kernel / series_scan_kernel scans (tad_kernels.cu: scan_grid)."""
    import torch
    B = 1 << logb
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    grid = max(1, min(-(-B // 1024), SCAN_MAX_CTAS, sms - 4))
    return -(-B // (grid * 1024)), sms


# --------------------------------------------------------------------------------------------------------------------
# 10^9 rows in passes
# --------------------------------------------------------------------------------------------------------------------
ORACLE_PIECE_ROWS = 100_000_000
ORACLE_WORKERS = 3
ORACLE_HOST_BYTES = 45e9           # the oracle's working set, three 10^8-row pieces at once: 32 GB measured, plus room
OPT_IN_1E9 = "TAD_TEST_WHOLE_1E9"


def _peak_rss():
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024


def test_1e9_rows_in_passes_every_row():
    """configs[2]'s shape (10^9 rows, 10^7 connections x 100) from pinned host columns, no memory budget: more than the
    device holds, so the job runs in passes.  The oracle runs first, in 10^8-row pieces by source address, and frees
    its device memory before the job starts; the free-HBM skip below is what makes sure the job has the device to
    itself otherwise.  The oracle takes minutes on this table: the test runs only on request."""
    import torch
    from theia_b200.engine import TadEngine
    if os.environ.get(OPT_IN_1E9) != "1":
        pytest.skip("the 10^9-row whole-table check takes minutes of oracle time; set %s=1 to run it" % OPT_IN_1E9)
    S, n = 10_000_000, 100
    R = S * n
    table_bytes = R * sum(np.dtype(d).itemsize for d in synth.COLUMN_DTYPES.values())
    if _mem_available() < 64e9:
        pytest.skip("needs ~64 GB of available host memory")
    if _mem_available() < table_bytes + ORACLE_HOST_BYTES:
        pytest.skip("the oracle's working set (~%.0f GB) does not fit in host memory next to the %.0f GB table" % (
            ORACLE_HOST_BYTES / 1e9, table_bytes / 1e9))
    torch.cuda.empty_cache()
    if torch.cuda.mem_get_info()[0] < 70e9:
        pytest.skip("needs ~70 GB of free HBM")
    with TadEngine(device=0) as e:
        cols = e.alloc_columns(R)
        try:
            synth.fill_columns_blocks(cols, S, n, seed=71, device=_cuda())
            table = {k: cols.view(k)[:R] for k in synth.COLUMN_DTYPES}
            rss0 = _peak_rss()
            t0 = time.perf_counter()
            want = co.run_job(table, algo=co.ALGO_EWMA, sort_device=_cuda(), max_chunk_rows=ORACLE_PIECE_ROWS,
                               workers=ORACLE_WORKERS)
            oracle_s = time.perf_counter() - t0
            oracle_peak = _peak_rss() - rss0
            torch.cuda.empty_cache()
            got, st, engine_s = run_engine(e, cols, algo="EWMA")
            report("1e9 EWMA in passes", engine_s, oracle_s, st,
                   peak_rss_gb="%.1f with the table, %.1f above it during the oracle" % (_peak_rss() / 1e9,
                                                                                          oracle_peak / 1e9))
            assert st["passes"] >= 2 and st["rows_in"] == R
            check_rows(got, st, want, "1e9 rows in passes")
        finally:
            cols.free()


# --------------------------------------------------------------------------------------------------------------------
# configs[1]: 10^8 rows, 10^6 connections x 100 points
# --------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def configs1():
    """The table on the device, the engine's view of it and the oracle's result per algorithm (computed once)."""
    import torch
    from theia_b200.engine import DeviceColumns
    torch.cuda.empty_cache()
    if torch.cuda.mem_get_info()[0] < 40e9:
        pytest.skip("needs ~40 GB of free HBM")
    S, n = 1_000_000, 100
    cols_t = synth.make_flows_torch(S, n, seed=7, device=_cuda())
    dcols = DeviceColumns(S * n, {k: v.data_ptr() for k, v in cols_t.items()})
    dcols.keepalive = cols_t
    host = synth.torch_cols_to_numpy(cols_t)
    want = {}

    def oracle(algo):
        if algo not in want:
            want[algo] = run_oracle(host, algo)
        return want[algo]
    yield dcols, oracle
    del dcols, cols_t, host, want
    torch.cuda.empty_cache()


@pytest.mark.parametrize("algo", ["EWMA", "DBSCAN"])
def test_configs1_every_row(engine, configs1, algo):
    dcols, oracle = configs1
    got, st, engine_s = run_engine(engine, dcols, algo=algo)
    want, oracle_s = oracle(algo)
    report("configs[1] %s" % algo, engine_s, oracle_s, st)
    assert st["rows_in"] == st["rows_kept"] == 100_000_000 and st["result_rows"] > 0
    check_rows(got, st, want, "configs[1] %s" % algo)


@pytest.mark.parametrize("logb", [18, 20, 22])
def test_configs1_buckets_past_one_per_scan_thread(configs1, logb):
    """2^logb buckets: each scan thread loops over several buckets (``per``, as scan_grid sizes the grid on this device;
    test_lumpy_buckets_past_one_per_scan_thread observes the bucket count the engine used); at 2^22 most buckets hold
    0 to 60 rows, the smallest capacity class, with long runs of empty buckets between series."""
    dcols, oracle = configs1
    per, sms = scan_per(logb)
    eng = make_engine(TAD_DEBUG_LOGB=str(logb))
    try:
        for algo in ("EWMA", "DBSCAN"):
            got, st, engine_s = run_engine(eng, dcols, algo=algo)
            want, oracle_s = oracle(algo)
            report("configs[1] %s at 2^%d buckets" % (algo, logb), engine_s, oracle_s, st, per=per, sms=sms)
            check_rows(got, st, want, "configs[1] %s logB %d" % (algo, logb))
    finally:
        eng.close()


def test_small_table_at_2_22_buckets():
    """10^5 rows over 2^22 buckets: one bucket in 2,000 holds a row, so almost every scan thread's buckets are empty
    and the series hint table spans long empty runs."""
    t = synth.make_flows(2000, 50, seed=91, ragged=True, dup_frac=0.05)
    eng = make_engine(TAD_DEBUG_LOGB="22")
    try:
        for algo in ("EWMA", "DBSCAN"):
            for kw in ({}, {"emit_all": True}, {"reducer": 1, "emit_all": True}):
                t0 = time.perf_counter()
                got, st = eng.run(t, algo=algo, tad_id="sparse", **kw)
                engine_s = time.perf_counter() - t0
                t0 = time.perf_counter()
                want, ns, npts = oracle_rows(t, algo, **kw)
                report("1e5 rows at 2^22 buckets %s %s (C oracle)" % (algo, kw), engine_s, time.perf_counter() - t0, st)
                assert (st["series"], st["points"], st["result_rows"]) == (ns, npts, len(want["flow_end"])), (kw, st)
                assert_same_rows(got, want, what="2^22 buckets, %s %s" % (algo, kw))
    finally:
        eng.close()


# --------------------------------------------------------------------------------------------------------------------
# a lumpy table
# --------------------------------------------------------------------------------------------------------------------
def lumpy_table(scale, seed):
    """About 10^8 * scale rows from make_flows pieces with 5 % duplicate rows: series of 1..5999 points, 6000-point
    series, 1..49-point series, and 1..39-point series with values within 1e10 of 2^64 - 1."""
    parts = [synth.make_flows(int(10_000 * scale), 3000, seed=seed, ragged=True, dup_frac=0.05),
             synth.make_flows(int(300 * scale), 6000, seed=seed + 1, dup_frac=0.05),
             synth.make_flows(int(2_600_000 * scale), 25, seed=seed + 2, ragged=True, dup_frac=0.05)]
    top = synth.make_flows(int(200_000 * scale), 20, seed=seed + 3, ragged=True, dup_frac=0.05)
    top["value"] = np.uint64(U64_MAX) - top["value"]
    parts.append(top)
    return {c: np.concatenate([p[c] for p in parts]) for c in synth.COLUMN_DTYPES}


def big_buckets(h, logb=None):
    """(buckets past the shared-memory capacity, their rows) of the rows with key hashes ``h`` at 2^logb buckets, by
    default the count the engine picks for that many rows."""
    logb = sharding.pick_logb(len(h)) if logb is None else logb
    hist = np.bincount((h >> np.uint64(64 - logb)).astype(np.int64), minlength=1 << logb)
    big = hist > GROUP_CAP
    return int(big.sum()), int(hist[big].sum())


@pytest.fixture(scope="module")
def lumpy(engine):
    import torch
    torch.cuda.empty_cache()
    if torch.cuda.mem_get_info()[0] < 40e9:
        pytest.skip("needs ~40 GB of free HBM")
    t = lumpy_table(1.0, seed=101)
    cols = engine.columns_from_numpy(t)
    want = {}

    def oracle(algo, reducer):
        if (algo, reducer) not in want:
            want[algo, reducer] = run_oracle(t, algo, reducer=reducer)
        return want[algo, reducer]
    yield t, cols, oracle, sharding.key_hash(t)
    cols.free()


@pytest.mark.parametrize("algo,reducer", [("EWMA", 0), ("EWMA", 1), ("DBSCAN", 0)])
def test_lumpy_table(engine, lumpy, algo, reducer):
    t, cols, oracle, h = lumpy
    got, st, engine_s = run_engine(engine, cols, algo=algo, reducer=reducer)
    want, oracle_s = oracle(algo, reducer)
    n_big, big_rows = big_buckets(h)
    report("lumpy 1e8 %s reducer %d" % (algo, reducer), engine_s, oracle_s, st, big_buckets=n_big)
    assert st["rows_in"] == len(t["flow_end"]) and st["points"] < st["rows_in"]
    check_rows(got, st, want, "lumpy %s reducer %d" % (algo, reducer))
    assert n_big >= 1000 and st["spill_rows"] == big_rows, (n_big, big_rows, st["spill_rows"])


@pytest.mark.parametrize("logb", [18, 20, 22])
def test_lumpy_buckets_past_one_per_scan_thread(lumpy, logb):
    """The lumpy table at 2^logb buckets.  The rows in buckets past 4,096 rows depend on the bucket count, and the
    engine's spill rows must equal the host's count at 2^logb -- which they cannot at any other bucket count tried
    here -- so the test sees that the engine ran with 2^logb buckets, and the scan threads with ``per`` each."""
    t, cols, oracle, h = lumpy
    counts = {b: big_buckets(h, b) for b in (18, 20, 22)}
    assert len({rows for _, rows in counts.values()}) == len(counts), counts
    per, sms = scan_per(logb)
    eng = make_engine(TAD_DEBUG_LOGB=str(logb))
    try:
        for algo in ("EWMA", "DBSCAN"):
            got, st, engine_s = run_engine(eng, cols, algo=algo)
            want, oracle_s = oracle(algo, 0)
            report("lumpy 1e8 %s at 2^%d buckets" % (algo, logb), engine_s, oracle_s, st, big_buckets=counts[logb][0],
                   per=per, sms=sms)
            check_rows(got, st, want, "lumpy %s logB %d" % (algo, logb))
            assert st["spill_rows"] == counts[logb][1], (logb, st["spill_rows"], counts)
    finally:
        eng.close()


@pytest.mark.parametrize("algo", ["EWMA", "DBSCAN"])
def test_lumpy_emit_all(engine, algo):
    """Every point of a 10^7-row lumpy table comes out, with its flag."""
    t = lumpy_table(0.1, seed=202)
    cols = engine.columns_from_numpy(t)
    try:
        got, st, engine_s = run_engine(engine, cols, algo=algo, reducer=1, emit_all=True)
    finally:
        cols.free()
    want, oracle_s = run_oracle(t, algo, reducer=1, emit_all=True)
    report("lumpy 1e7 %s emit_all" % algo, engine_s, oracle_s, st)
    assert st["result_rows"] == st["points"] > 9_000_000
    check_rows(got, st, want, "lumpy emit_all %s" % algo)


def wide_lumpy_table(scale, seed):
    """A lumpy table whose series are three in four drawn uniformly from [1, 10^13): values 40,000 eps apart on
    average, so DBSCAN finds most of their points noise."""
    t = lumpy_table(scale, seed)
    rng = np.random.default_rng(seed)
    wide = (t["src_ip"] & np.uint32(3)) != 0
    t["value"] = np.where(wide, rng.integers(1, 10 ** 13, len(wide), dtype=np.uint64), t["value"]).astype(np.uint64)
    return t


@pytest.mark.parametrize("algo", ["EWMA", "DBSCAN"])
def test_result_capacity_rerun(engine, algo):
    """Without emit_all, detect first writes into room for rows / 8 + 65536 results (tad_engine.cu: out_cap_guess, from
    the kept rows for EWMA and the points for DBSCAN).  Here more points are flagged than that, so detect runs again
    with the exact count and writes millions of rows; every one must equal the oracle's.  EWMA flags that many on the
    lumpy table itself (the EWMA climbs from 0 through the first points of every near-constant series); DBSCAN on the
    table with values spread far beyond eps."""
    t = lumpy_table(0.1, seed=303) if algo == "EWMA" else wide_lumpy_table(0.1, seed=303)
    cols = engine.columns_from_numpy(t)
    try:
        got, st, engine_s = run_engine(engine, cols, algo=algo)
    finally:
        cols.free()
    want, oracle_s = run_oracle(t, algo)
    report("result-capacity rerun 1e7 %s" % algo, engine_s, oracle_s, st)
    assert st["result_rows"] > st["rows_kept"] // 8 + 65536 > 1_000_000, st
    check_rows(got, st, want, "result-capacity rerun %s" % algo)
