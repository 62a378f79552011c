"""Parity of the partition scatter's less common paths with the oracle, bit-exact on every column.  The scatter writes each
row from a lane pair, so every table here ends in a partially filled warp and in a partial group of eight rows: a row
whose pair did not take part in the store would leave a stale slot, which shows up as a foreign or missing result row."""
import os

import numpy as np
import pytest

from theia_b200 import synth
from tests.util import assert_same_rows, oracle_rows

pytestmark = pytest.mark.gpu

_SIGNED = {np.dtype(np.uint32): np.int32, np.dtype(np.uint16): np.int16, np.dtype(np.uint64): np.int64,
           np.dtype(np.uint8): np.uint8}


def _ends_in_partial_warp(rows):
    groups = (rows + 7) // 8              # eight rows per lane
    return rows % 8 != 0 and groups % 32 != 0


def _run(engine, cols, table, emit_all=True):
    job = engine.submit(cols, algo="EWMA", tad_id="scatter", emit_all=emit_all)
    try:
        st = job.wait()
        got = job.result()
    finally:
        job.release()
        cols.free()
    want, ns, npts = oracle_rows(table, "EWMA", emit_all=emit_all)
    assert st["state"] == "COMPLETED"
    assert st["series"] == ns and st["points"] == npts, (st, ns, npts)
    assert_same_rows(got, want, what="rows %d" % len(table["flow_end"]))


def _unaligned_device_cols(table):
    """Device-resident columns that each start one element past an allocation: none is 16-byte aligned, so the scatter
    takes its scalar-load instance."""
    import torch
    from theia_b200.engine import DeviceColumns
    bufs = {}
    for k, v in table.items():
        t = torch.from_numpy(np.ascontiguousarray(v).view(_SIGNED[v.dtype])).cuda()
        buf = torch.zeros(len(t) + 1, dtype=t.dtype, device=t.device)
        buf[1:] = t
        bufs[k] = buf
    ptrs = {k: b[1:].data_ptr() for k, b in bufs.items()}
    assert all(p % 16 for p in ptrs.values())
    d = DeviceColumns(len(table["flow_end"]), ptrs)
    d.keepalive = bufs
    return d


@pytest.fixture(scope="module")
def exact_engine():
    """Engine that always runs the exact partition (histogram + scan + scatter at absolute cursors)."""
    from theia_b200.engine import TadEngine
    os.environ["TAD_OPTIMISTIC"] = "0"
    try:
        eng = TadEngine(device=0)
    finally:
        del os.environ["TAD_OPTIMISTIC"]
    yield eng
    eng.close()


@pytest.mark.parametrize("emit_all", [False, True])
def test_second_grid_stride_ends_in_partial_warp(engine, emit_all):
    """2,163,103 rows = 270,388 groups of eight, not a multiple of 32: more than one grid of at most 8 CTAs of 256 lanes
    per SM covers, so the last grid-stride iteration ends in a partial warp."""
    t = synth.make_flows(21001, 103, seed=51)
    rows = len(t["flow_end"])
    assert (rows + 7) // 8 > 132 * 8 * 256 and _ends_in_partial_warp(rows)
    _run(engine, engine.columns_from_numpy(t), t, emit_all=emit_all)


def test_unaligned_columns_and_exact_partition(engine, exact_engine):
    """One table through the scalar-load scatter (unaligned device columns) on the optimistic partition, then through the
    exact partition from host and from unaligned device columns.  A larger table runs first on the exact engine, so that
    an unwritten row of the second would read a row of the first."""
    t = synth.make_flows(3001, 37, seed=52)
    rows = len(t["flow_end"])
    assert _ends_in_partial_warp(rows)
    _run(engine, _unaligned_device_cols(t), t)
    big = synth.make_flows(5000, 40, seed=53)
    _run(exact_engine, exact_engine.columns_from_numpy(big), big)
    _run(exact_engine, exact_engine.columns_from_numpy(t), t)
    _run(exact_engine, _unaligned_device_cols(t), t)
