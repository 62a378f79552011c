"""EWMA scored inside the group kernel: every result column bit-exact against the oracle, and the series / point counts
equal to the oracle's, on the paths around the fused kernel (result-capacity rerun, every shared-memory capacity class,
buckets that spill next to buckets that are scored in place, duplicate reduction with both reducers)."""
import os

import numpy as np
import pytest

from theia_b200 import synth
from tests.util import assert_same_rows, oracle_rows

pytestmark = pytest.mark.gpu


def make_engine(**env):
    """An engine created under the given environment (read once, when the context is created)."""
    from theia_b200.engine import TadEngine
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return TadEngine(device=0)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def exact_engine():
    """The exact partition: the group kernel reads the rows straight out of part[], where other kernels write series
    entries in place, so a rerun that read overwritten rows would give wrong keys."""
    eng = make_engine(TAD_OPTIMISTIC="0")
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def engine16():
    """16 hash buckets: the table size alone picks the capacity class (and the spill) of every bucket."""
    eng = make_engine(TAD_DEBUG_LOGB="4")
    yield eng
    eng.close()


def check(engine, table, **kw):
    got, st = engine.run(table, algo="EWMA", tad_id="fused", **kw)
    want, ns, npts = oracle_rows(table, "EWMA", **kw)
    assert st["state"] == "COMPLETED"
    assert st["series"] == ns and st["points"] == npts, (st, ns, npts)
    assert st["result_rows"] == len(want["flow_end"])
    assert_same_rows(got, want, what="fused EWMA %s" % (kw,))
    return got, st


@pytest.mark.parametrize("which", ["default", "exact"])
def test_result_capacity_rerun(engine, exact_engine, which):
    """Four points per series of nearly constant values: every point is flagged (the EWMA starts at 0 and is still far
    below the values), far more rows than the first capacity guess, so the group kernel runs a second time."""
    t = synth.make_flows(60_000, 4, seed=41)
    rows = len(t["value"])
    got, st = check(engine if which == "default" else exact_engine, t)
    assert st["result_rows"] > rows // 8 + 65536


@pytest.mark.parametrize("rows_per_bucket", [700, 1500, 3000])
@pytest.mark.parametrize("points", [1, 20])
def test_capacity_classes(engine16, rows_per_bucket, points):
    """Buckets of about 700, 1500 and 3000 rows take the 1024-, 2048- and 4096-row instances; one-point series make a
    bucket of as many series as rows."""
    t = synth.make_flows(16 * rows_per_bucket // points, points, seed=42 + rows_per_bucket + points)
    got, st = check(engine16, t, emit_all=True)
    assert st["spill_rows"] == 0
    check(engine16, t)


def test_spilled_and_fused_buckets(engine16):
    """Three 5000-point connections overfill their buckets and take the spill path; the rest of the table is scored in
    place.  Every series is scored exactly once: the counts and the rows match the oracle."""
    t1 = synth.make_flows(3, 5000, seed=43, dup_frac=0.05)
    t2 = synth.make_flows(1500, 20, seed=44, ragged=True)
    t = {k: np.concatenate([t1[k], t2[k]]) for k in t1}
    got, st = check(engine16, t, emit_all=True)
    assert 15000 <= st["spill_rows"] < st["rows_kept"]
    check(engine16, t)


@pytest.mark.parametrize("reducer", [0, 1])
@pytest.mark.parametrize("emit_all", [False, True])
def test_duplicates(engine, reducer, emit_all):
    """(key, flowEndSeconds) duplicates are reduced with max or sum before scoring."""
    t = synth.make_flows(4000, 30, seed=45, dup_frac=0.3, ragged=True)
    check(engine, t, reducer=reducer, emit_all=emit_all)
