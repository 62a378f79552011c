"""The group kernel's finer capacity classes (512, 768 and 1280 rows) at their boundaries, and a bucket that fills every
class's hash table: a table whose 16 hash buckets hold exactly the row counts below (chosen through the host mirror of the
key hash).  With one point per connection the buckets of 512, 768, 1024, 1280, 1536, 2048 and 4096 rows hold as many
distinct keys as their class has rows, the highest load the 1.5-slots-per-row hash table sees.  EWMA (scored inside the
group kernel) and DBSCAN are compared bit for bit against the C oracle; ARIMA, whose group instance writes the per-series
arrays without value ranks, is checked on its series and point counts and on every column its fit does not compute."""
import numpy as np
import pytest

from theia_b200 import sharding, synth
from tests.test_gpu_group_detect import make_engine
from tests.util import assert_same_rows, oracle_rows

LOGB = 4
# rows of bucket b: both sides of the 512-, 768- and 1280-row capacities, every class's capacity exactly, a small and a
# one-row bucket, and an empty one
SIZES = [511, 512, 513, 767, 768, 769, 1024, 1279, 1280, 1281, 1536, 2048, 4096, 100, 1, 0]
KEY_COLS = ("src_ip", "dst_ip", "src_port", "dst_port", "proto", "flow_start")


@pytest.fixture(scope="module")
def engine16():
    eng = make_engine(TAD_DEBUG_LOGB=str(LOGB))
    yield eng
    eng.close()


def boundary_table(points, seed, dup_frac=0.0):
    """Rows of a synthetic table drawn bucket by bucket until bucket b holds exactly SIZES[b] rows."""
    pool = synth.make_flows(140_000 // points, points, seed=seed, dup_frac=dup_frac)
    bucket = sharding.key_hash(pool) >> np.uint64(64 - LOGB)
    pick = []
    for b, n in enumerate(SIZES):
        rows = np.flatnonzero(bucket == b)
        assert len(rows) >= n, (b, len(rows), n)
        pick.append(rows[:n])
    pick = np.random.default_rng(seed).permutation(np.concatenate(pick))
    return {k: v[pick] for k, v in pool.items()}


def check(engine, table, algo="EWMA", **kw):
    got, st = engine.run(table, algo=algo, tad_id="fineclasses", **kw)
    want, ns, npts = oracle_rows(table, algo, **kw)
    assert st["state"] == "COMPLETED"
    assert st["spill_rows"] == 0
    assert st["series"] == ns and st["points"] == npts, (st, ns, npts)
    assert st["result_rows"] == len(want["flow_end"])
    assert_same_rows(got, want, what="%s %s" % (algo, kw))


def test_bucket_sizes():
    """The table builder gives every bucket its planned row count, and the one-point table as many keys as rows (host
    only)."""
    for points in (1, 20):
        t = boundary_table(points, seed=90 + points)
        got = np.bincount((sharding.key_hash(t) >> np.uint64(64 - LOGB)).astype(np.int64), minlength=1 << LOGB)
        assert got.tolist() == SIZES
    keys = set(zip(*(t1.tolist() for t1 in (boundary_table(1, seed=91)[c] for c in KEY_COLS))))
    assert len(keys) == sum(SIZES)


@pytest.mark.gpu
@pytest.mark.parametrize("emit_all", [False, True])
@pytest.mark.parametrize("points", [1, 20])
def test_ewma_fine_class_boundaries(engine16, points, emit_all):
    check(engine16, boundary_table(points, seed=90 + points), emit_all=emit_all)


@pytest.mark.gpu
@pytest.mark.parametrize("emit_all", [False, True])
@pytest.mark.parametrize("reducer", [0, 1])
def test_duplicates_at_fine_class_boundaries(engine16, reducer, emit_all):
    """(key, flowEndSeconds) duplicates, reduced with max or sum before scoring, in one-point and in 20-point series."""
    for points in (1, 20):
        check(engine16, boundary_table(points, seed=100 + points, dup_frac=0.3), reducer=reducer, emit_all=emit_all)


@pytest.mark.gpu
@pytest.mark.parametrize("points", [1, 20])
def test_dbscan_fine_class_boundaries(engine16, points):
    check(engine16, boundary_table(points, seed=110 + points, dup_frac=0.1), algo="DBSCAN", emit_all=True)


@pytest.mark.gpu
def test_arima_fine_class_boundaries(engine16):
    """ARIMA emits every point of a series it fits and none of one it cannot; the rows it emits carry the same keys, times,
    values and stddev_samp as the oracle's rows of those series."""
    table = boundary_table(20, seed=120, dup_frac=0.1)
    got, st = engine16.run(table, algo="ARIMA", tad_id="fineclasses", emit_all=True)
    want, ns, npts = oracle_rows(table, "EWMA", emit_all=True)
    assert st["state"] == "COMPLETED"
    assert st["spill_rows"] == 0
    assert st["series"] == ns and st["points"] == npts, (st, ns, npts)
    assert len(got["flow_end"]) > 0
    fitted = set(zip(*(np.asarray(got[c]).tolist() for c in KEY_COLS)))
    keep = np.array([k in fitted for k in zip(*(want[c].tolist() for c in KEY_COLS))], dtype=bool)
    want = {c: np.asarray(v)[keep] for c, v in want.items()}
    got = {c: np.asarray(v) for c, v in got.items()}
    assert len(got["flow_end"]) == len(want["flow_end"])
    order_g = np.lexsort([got[k] for k in ("flow_end",) + KEY_COLS])
    order_w = np.lexsort([want[k] for k in ("flow_end",) + KEY_COLS])
    for c in KEY_COLS + ("flow_end", "throughput", "stddev"):
        assert np.array_equal(got[c][order_g], want[c][order_w], equal_nan=c == "stddev"), "ARIMA: column %s differs" % c
