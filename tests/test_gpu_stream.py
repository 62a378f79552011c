"""Streamed input (tad_submit_stream / tad_stream_push / tad_stream_end): the rows of a job arrive as column blocks,
round after round while the engine needs them again.  Every result equals a one-shot tad_submit of the whole table bit
for bit, on all 11 result columns and on the status counters, whatever the block sizes, memory kinds and row order."""
import os
import shutil
import subprocess
import time

import numpy as np
import pytest

from theia_b200 import synth
from tests.util import assert_same_rows, oracle_rows

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MB = 1 << 20
BUDGET_2 = 150 * MB
BUDGET_4 = 64 * MB
COUNTS = ("rows_in", "rows_kept", "points", "series", "result_rows")
_SIGNED = {np.dtype(np.uint32): np.int32, np.dtype(np.uint16): np.int16, np.dtype(np.uint64): np.int64,
           np.dtype(np.uint8): np.uint8}
ERR_INVALID_ARG, ERR_STATE, ERR_CANCELLED = -1, -5, -6


@pytest.fixture(scope="module")
def eng():
    """A context of its own: the budgets set here must not reach the session's engine."""
    from theia_b200.engine import TadEngine
    e = TadEngine(device=0)
    yield e
    e.close()


def _cuts(n, sizes, seed):
    if sizes == "whole":
        return [0, n]
    if sizes == "uneven":
        rng = np.random.default_rng(seed)
        cuts = [0]
        while cuts[-1] < n:
            cuts.append(min(n, cuts[-1] + int(rng.choice([1, 7, 2047, 4096, 30000, 65536]))))
        return cuts
    return list(range(0, n, sizes)) + [n]


def block_source(eng, table, sizes, kind):
    """blocks_factory for run_stream: every round in its own row order, cut into `sizes`, from pageable numpy arrays,
    two alternating pinned buffers, or device memory."""
    rounds = [0]
    n = len(table["flow_end"])
    pinned = []

    def factory():
        r = rounds[0]
        rounds[0] += 1
        perm = np.random.default_rng(1000 + r).permutation(n)
        t = {k: v[perm] for k, v in table.items()}
        cuts = _cuts(n, sizes, r)
        for k, (lo, hi) in enumerate(zip(cuts[:-1], cuts[1:])):
            part = {c: v[lo:hi] for c, v in t.items()}
            if kind == "pageable":
                yield part
            elif kind == "pinned":
                if not pinned:
                    cap = max(b - a for a, b in zip(cuts[:-1], cuts[1:]))
                    pinned.extend(eng.alloc_columns(max(cap, 65536)) for _ in range(2))
                yield pinned[k & 1].fill(part)      # buffer k & 1 is free again: push k-1 has returned
            else:
                yield device_cols(part)
    factory.free = lambda: [c.free() for c in pinned]
    return factory


def device_cols(table):
    import torch
    from theia_b200.engine import DeviceColumns
    ts = {k: torch.from_numpy(np.ascontiguousarray(v).view(_SIGNED[v.dtype])).cuda() for k, v in table.items()
          if v is not None and k not in ("src_ns", "dst_ns")}
    torch.cuda.synchronize()              # the engine's stream does not wait for torch's
    d = DeviceColumns(len(table["flow_end"]), {k: t.data_ptr() for k, t in ts.items()})
    d.keepalive = ts
    return d


def one_shot(eng, table, budget=0, **kw):
    eng.set_memory_budget(budget)
    return eng.run(table, tad_id="one-shot", **kw)


def streamed(eng, table, sizes, kind, budget=0, **kw):
    eng.set_memory_budget(budget)
    factory = block_source(eng, table, sizes, kind)
    try:
        return eng.run_stream(factory, tad_id="stream", **kw)
    finally:
        factory.free()


def same(got, st, ref, st_ref, what):
    for k in COUNTS:
        assert st[k] == st_ref[k], (what, k, st[k], st_ref[k])
    assert_same_rows(got, ref, what=what)


TABLE = synth.make_flows(300, 40, seed=81, dup_frac=0.25)


@pytest.mark.parametrize("algo", ["EWMA", "DBSCAN"])
@pytest.mark.parametrize("sizes,kind", [(1, "pinned"), (2047, "pageable"), (65536, "pinned"), ("uneven", "device"),
                                        ("whole", "pageable"), (2047, "device"), ("uneven", "pinned")])
def test_parity_with_one_shot(eng, algo, sizes, kind):
    ref, st_ref = one_shot(eng, TABLE, algo=algo, emit_all=True)
    got, st = streamed(eng, TABLE, sizes, kind, algo=algo, emit_all=True, rows_hint=len(TABLE["flow_end"]))
    assert st["rounds"] == 1 and st["memory"]["passes"] == 1 and st["state"] == "COMPLETED"
    same(got, st, ref, st_ref, "%s %s %s" % (algo, sizes, kind))
    want, ns, npts = oracle_rows(TABLE, algo, emit_all=True)
    assert st["series"] == ns and st["points"] == npts
    assert_same_rows(got, want, what="vs oracle")


@pytest.mark.parametrize("reducer", [0, 1])
@pytest.mark.parametrize("kind", ["pageable", "pinned"])
def test_filters_and_reducers(eng, reducer, kind):
    t = synth.make_flows(2000, 60, seed=82, dup_frac=0.3)
    rng = np.random.default_rng(82)
    n = len(t["value"])
    t["src_ns"] = rng.integers(0, 6, n).astype(np.uint32)
    t["dst_ns"] = rng.integers(0, 6, n).astype(np.uint32)
    kw = dict(reducer=reducer, start_time=synth.T0 + 600, end_time=synth.T0 + 3000, ns_ignore=(1, 4), emit_all=True)
    ref, st_ref = one_shot(eng, t, **kw)
    got, st = streamed(eng, t, "uneven", kind, **kw)
    assert st["rows_kept"] < st["rows_in"] == n
    same(got, st, ref, st_ref, "filters reducer=%d %s" % (reducer, kind))
    keep = ~np.isin(t["src_ns"], (1, 4)) & ~np.isin(t["dst_ns"], (1, 4))
    want, _, _ = oracle_rows({k: v[keep] for k, v in t.items() if k not in ("src_ns", "dst_ns")}, "EWMA", reducer=reducer,
                             start_time=synth.T0 + 600, end_time=synth.T0 + 3000, emit_all=True)
    assert_same_rows(got, want, what="filters vs oracle")


def test_arima_small_table(eng):
    t = synth.make_flows(60, 30, seed=83, dup_frac=0.1)
    ref, st_ref = one_shot(eng, t, algo="ARIMA", emit_all=True)
    got, st = streamed(eng, t, 97, "pageable", algo="ARIMA", emit_all=True)
    same(got, st, ref, st_ref, "ARIMA")


BIG = synth.make_flows(20000, 100, seed=84)           # 2M rows


@pytest.mark.parametrize("kind,budget,min_passes", [("pinned", BUDGET_2, 2), ("pinned", BUDGET_4, 4),
                                                    ("device", BUDGET_2, 2), ("device", BUDGET_4, 4)])
def test_rounds_under_a_budget(eng, kind, budget, min_passes):
    ref, st_ref = one_shot(eng, BIG)
    n = len(BIG["flow_end"])
    got, st = streamed(eng, BIG, 65536, kind, budget=budget, rows_hint=n)
    mem = st["memory"]
    assert st["rounds"] == mem["passes"] >= min_passes, (st["rounds"], mem)
    assert mem["peak_workspace_bytes"] <= budget, mem
    same(got, st, ref, st_ref, "budget %d %s" % (budget, kind))
    got0, st0 = streamed(eng, BIG, "uneven", kind, budget=budget, rows_hint=0)
    assert st0["rounds"] <= st["rounds"] + 1, (st0["rounds"], st["rounds"])
    same(got0, st0, ref, st_ref, "budget %d %s, no hint" % (budget, kind))


@pytest.mark.parametrize("budget,factor", [(0, 10 ** 6), (BUDGET_2, 8)])
def test_overestimated_hint_costs_at_most_one_round(eng, budget, factor):
    """A hint far above the real row count must not cost a round for every surplus pass: the planner falls back to the
    pass count the first round's rows call for."""
    ref, st_ref = one_shot(eng, BIG)
    n = len(BIG["flow_end"])
    _, st_exact = streamed(eng, BIG, 65536, "pinned", budget=budget, rows_hint=n)
    got, st = streamed(eng, BIG, 65536, "pinned", budget=budget, rows_hint=factor * n)
    assert st["rounds"] <= st_exact["rounds"] + 1, (st["rounds"], st_exact["rounds"])
    assert st["memory"]["passes"] == st_exact["memory"]["passes"]
    same(got, st, ref, st_ref, "hint x%d budget %d" % (factor, budget))


@pytest.mark.parametrize("kind", ["pinned", "device"])
def test_pass_columns_grow_without_a_hint(eng, kind):
    """No hint, no budget, 3M rows: the pass columns start at 1M rows and grow twice while the round arrives, carrying the
    rows they hold; the one pass then runs on them."""
    t = synth.make_flows(30000, 100, seed=92, dup_frac=0.1)
    ref, st_ref = one_shot(eng, t, emit_all=True)
    got, st = streamed(eng, t, 65536, kind, rows_hint=0, emit_all=True)
    assert st["rounds"] == 1 and st["memory"]["passes"] == 1
    same(got, st, ref, st_ref, "growth %s" % kind)


def test_spill_inside_a_streamed_pass(eng):
    small = synth.make_flows(20000, 100, seed=85)
    big = synth.make_flows(30, 6000, seed=86)
    t = {k: np.concatenate([small[k], big[k]]) for k in small}
    ref, st_ref = one_shot(eng, t, emit_all=True)
    got, st = streamed(eng, t, 65536, "pinned", budget=BUDGET_4, rows_hint=len(t["flow_end"]), emit_all=True)
    assert st["spill_rows"] > 0 and st["memory"]["passes"] >= 4
    same(got, st, ref, st_ref, "spill")


def _normal_job_ok(eng):
    t = synth.make_flows(200, 30, seed=87)
    got, _ = one_shot(eng, t, emit_all=True)
    want, _, _ = oracle_rows(t, "EWMA", emit_all=True)
    assert_same_rows(got, want, what="normal job after a protocol error")


def _code(excinfo):
    return excinfo.value.code


def test_round_that_omits_a_block_fails(eng):
    from theia_b200.engine import TadError
    eng.set_memory_budget(BUDGET_2)
    factory = block_source(eng, BIG, 65536, "pinned")
    job = eng.submit_stream(rows_hint=len(BIG["flow_end"]), tad_id="omit")
    try:
        for b in factory():
            job.push(b)
        assert job.end()                        # needs another round
        with pytest.raises(TadError) as e:
            for i, b in enumerate(factory()):
                if i != 3:
                    job.push(b)
            job.end()
        assert _code(e) == ERR_INVALID_ARG
        st = job.wait(check=False)
        assert st["state"] == "FAILED" and "changed" in st["err_msg"], st["err_msg"]
    finally:
        job.release()
        factory.free()
    _normal_job_ok(eng)


def test_protocol_errors(eng):
    from theia_b200.engine import TadError
    eng.set_memory_budget(0)
    t = synth.make_flows(100, 20, seed=88)
    half = {k: v[:1000] for k, v in t.items()}
    # a block with another column set
    job = eng.submit_stream(tad_id="cols")
    job.push(half)
    with pytest.raises(TadError) as e:
        job.push({k: v for k, v in half.items() if k != "src_port"})
    assert _code(e) == ERR_INVALID_ARG
    assert job.wait(check=False)["state"] == "FAILED"
    job.release()
    _normal_job_ok(eng)
    # push after the input is complete
    job = eng.submit_stream(tad_id="late")
    job.push(half)
    assert job.end() is False
    with pytest.raises(TadError) as e:
        job.push(half)
    assert _code(e) == ERR_STATE
    with pytest.raises(TadError) as e:
        job.end()
    assert _code(e) == ERR_STATE
    assert job.wait()["state"] == "COMPLETED"
    job.release()
    # push and end on a tad_submit job
    cols = eng.columns_from_numpy(half)
    job = eng.submit(cols)
    import ctypes as C
    from theia_b200 import _lib as L
    assert eng.lib.tad_stream_push(job.h, C.byref(cols.c)) == ERR_STATE
    assert eng.lib.tad_stream_end(job.h, C.byref(C.c_int32())) == ERR_STATE
    job.wait()
    job.release()
    cols.free()
    assert L.TAD_MEM_HOST == 0
    _normal_job_ok(eng)


def test_cancel_mid_round(eng):
    from theia_b200.engine import TadError
    eng.set_memory_budget(0)
    t = synth.make_flows(100, 20, seed=89)
    job = eng.submit_stream(tad_id="cancel")
    job.push({k: v[:500] for k, v in t.items()})
    job.cancel()
    with pytest.raises(TadError) as e:
        job.push({k: v[500:] for k, v in t.items()})
    assert _code(e) == ERR_CANCELLED
    assert job.poll()["state"] == "FAILED"
    with pytest.raises(TadError) as e:
        job.end()
    assert _code(e) == ERR_CANCELLED
    job.release()
    _normal_job_ok(eng)


def test_release_without_end_is_prompt(eng):
    eng.set_memory_budget(0)
    t = synth.make_flows(100, 20, seed=90)
    job = eng.submit_stream(tad_id="release")
    job.push(t)
    time.sleep(0.2)                         # the worker has taken the block and waits for more
    t0 = time.perf_counter()
    job.release()
    assert time.perf_counter() - t0 < 2.0
    _normal_job_ok(eng)


def test_empty_stream(eng):
    eng.set_memory_budget(0)
    got, st = eng.run_stream(lambda: iter(()), tad_id="empty")
    assert st["state"] == "COMPLETED" and st["rounds"] == 1
    assert st["rows_in"] == st["result_rows"] == 0 and len(got["flow_end"]) == 0
    _normal_job_ok(eng)


def test_c_stream_example(tmp_path):
    """examples/tad_stream.c drives a streamed job from plain C and gets the result count of a one-shot tad_submit."""
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    exe = str(tmp_path / "tad_stream")
    subprocess.check_call([gcc, "-std=c99", "-Wall", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "examples", "tad_stream.c"), "-L", os.path.join(ROOT, "theia_b200"),
                           "-ltheia_tad", "-Wl,-rpath," + os.path.join(ROOT, "theia_b200"), "-o", exe])
    for args in ([], [str(64 * MB)]):
        out = subprocess.run([exe] + args, capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
        assert "same result count" in out.stdout and "300000 rows in" in out.stdout, out.stdout
        print(out.stdout)
