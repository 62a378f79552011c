"""The group kernel's shared-memory capacity classes at their boundaries: a table whose 16 hash buckets hold exactly the
row counts below (chosen through the host mirror of the key hash), so that buckets sit on both sides of every class
capacity.  Every result column is compared bit for bit against the C oracle, with EWMA scored inside the group kernel
and with DBSCAN, whose group instances write the per-series arrays instead."""
import numpy as np
import pytest

from theia_b200 import sharding, synth
from tests.test_gpu_group_detect import make_engine
from tests.util import assert_same_rows, oracle_rows

LOGB = 4
# rows of bucket b: both sides of the 1024-, 1536-, 2048- and 4096-row capacities, and an empty bucket
SIZES = [1000, 1024, 1025, 1100, 1500, 1536, 1537, 1600, 2000, 2048, 2049, 2100, 4000, 4096, 700, 0]


@pytest.fixture(scope="module")
def engine16():
    eng = make_engine(TAD_DEBUG_LOGB=str(LOGB))
    yield eng
    eng.close()


def boundary_table(points, seed, dup_frac=0.0):
    """Rows of a synthetic table drawn bucket by bucket until bucket b holds exactly SIZES[b] rows.  With one point per
    connection a bucket holds as many series as rows: the fullest its hash table gets."""
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
    got, st = engine.run(table, algo=algo, tad_id="classes", **kw)
    want, ns, npts = oracle_rows(table, algo, **kw)
    assert st["state"] == "COMPLETED"
    assert st["spill_rows"] == 0
    assert st["series"] == ns and st["points"] == npts, (st, ns, npts)
    assert st["result_rows"] == len(want["flow_end"])
    assert_same_rows(got, want, what="%s %s" % (algo, kw))


def test_bucket_sizes():
    """The table builder gives every bucket its planned row count (host only)."""
    t = boundary_table(20, seed=60)
    got = np.bincount((sharding.key_hash(t) >> np.uint64(64 - LOGB)).astype(np.int64), minlength=1 << LOGB)
    assert got.tolist() == SIZES


@pytest.mark.gpu
@pytest.mark.parametrize("emit_all", [False, True])
@pytest.mark.parametrize("points", [1, 20])
def test_ewma_class_boundaries(engine16, points, emit_all):
    check(engine16, boundary_table(points, seed=61 + points), emit_all=emit_all)


@pytest.mark.gpu
@pytest.mark.parametrize("emit_all", [False, True])
@pytest.mark.parametrize("reducer", [0, 1])
def test_duplicates_at_class_boundaries(engine16, reducer, emit_all):
    """(key, flowEndSeconds) duplicates, reduced with max or sum before scoring, in one-point and in 20-point series."""
    for points in (1, 20):
        check(engine16, boundary_table(points, seed=70 + points, dup_frac=0.3), reducer=reducer, emit_all=emit_all)


@pytest.mark.gpu
@pytest.mark.parametrize("points", [1, 20])
def test_dbscan_class_boundaries(engine16, points):
    check(engine16, boundary_table(points, seed=80 + points, dup_frac=0.1), algo="DBSCAN", emit_all=True)
