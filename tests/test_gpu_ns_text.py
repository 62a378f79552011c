"""The namespace ignore list tested on the GPU from namespace text (tad_submit_stream_filtered_ns, tad_stream_push_text_ns):
the result rows and counts equal, bit for bit, those of the same rows pushed with host namespace ids and the ignore list as
ids -- with text and with push-down u32 addresses, in one pass, in hash-range passes and with a host row store that holds
only the kept rows, and for a flagged job run in a fit yield or fitting beside a fit.  Bad namespace text fails with
TAD_ERR_INVALID_ARG and the context runs the next job.  The job entry point under TAD_DEVICE_NS=1 writes the INSERT body
of its host-encoded path in every mode."""
import threading
import time

import numpy as np
import pytest

from theia_b200 import anomaly_detection as ad
from theia_b200 import synth
from tests.util import assert_same_rows

from .test_gpu_fit_sharing import RESERVE, _device_table
from .test_gpu_job_entry_stream import HOST, _Recording, canonical_rows, same
from .test_gpu_stream import BIG, BUDGET_4, TABLE, _normal_job_ok
from .test_gpu_text_keys import name_of
from .test_job_entry_stream import TableTransport, make_table
from .test_text_keys import column_from_names, text_table

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG = -1
LONG_NS = b"ns-" + b"x" * 60                   # longer than the text staging's 48 bytes per row
NS = [b"default", b"kube-system", b"flow-visibility", b"", LONG_NS] + [b"team-%02d" % k for k in range(35)]
LISTS = [[], [b"kube-system"], [b"kube-system", b"flow-visibility", b"", LONG_NS, b"no-such-ns"]]


@pytest.fixture(scope="module")
def eng():
    """A context of its own: the budgets set here must not reach the session's engine."""
    from theia_b200.engine import TadEngine
    e = TadEngine(device=0)
    yield e
    e.close()


def _namespaces(n, seed):
    """Per row the source and destination namespace (indices into NS), about one row in six listed by LISTS[1]."""
    rng = np.random.default_rng(seed)
    p = np.full(len(NS), 0.7 / (len(NS) - 4))
    p[:4] = (0.1, 0.1, 0.05, 0.05)
    return rng.choice(len(NS), n, p=p / p.sum()), rng.choice(len(NS), n, p=p / p.sum())


def blocks(table, ns, cuts, ns_text, addr_text):
    """The table's rows in blocks: (columns, text) with the namespaces as text or as ids (their index in NS) and the
    addresses as text or as u32."""
    addr = {s: text_table(table[s], name_of) for s in ("src_ip", "dst_ip")} if addr_text else {}
    out = []
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        b = {k: v[lo:hi] for k, v in table.items()}
        txt = {}
        for s, (names, inv) in addr.items():
            txt[s] = column_from_names(names, inv[lo:hi])
            b[s] = None
        for s, idx in zip(("src_ns", "dst_ns"), ns):
            if ns_text:
                txt[s] = column_from_names(NS, idx[lo:hi])
            else:
                b[s] = idx[lo:hi].astype(np.uint32)
        out.append((b, txt))
    return out


def feed(job, bl):
    n, again = 0, True
    while again:
        for b, txt in bl:
            job.push(b, text=txt or None)
        again = job.end()
        n += 1
    return n


def _kw(names, ns_text):
    if ns_text:
        return {"ns_ignore_names": names}
    return {"ns_ignore": [NS.index(x) for x in names if x in NS]}


def _run(eng, bl, names, ns_text, budget=0, host=0, **kw):
    eng.set_memory_budget(budget)
    eng.set_host_budget(host)
    job = eng.submit_stream(tad_id="ns", **_kw(names, ns_text), **kw)
    try:
        rounds = feed(job, bl)
        st = job.wait()
        st["rounds"], st["memory"] = rounds, job.memory()
        return job.result(), st
    finally:
        job.release()
        eng.set_host_budget(0)
        eng.set_memory_budget(0)


def _check(eng, table, ns, cuts, names, addr_text, budget=0, host=0, **kw):
    ref, st_ref = _run(eng, blocks(table, ns, cuts, False, addr_text), names, False, budget, host, **kw)
    got, st = _run(eng, blocks(table, ns, cuts, True, addr_text), names, True, budget, host, **kw)
    for k in ("rows_in", "rows_kept", "points", "series", "result_rows"):
        assert st[k] == st_ref[k], (k, names)
    assert (st["rows_kept"] < st["rows_in"]) == bool(set(names) & set(NS)), names
    assert_same_rows(got, ref, what="namespace text vs ids %r" % (names,))
    return st


def _cuts(n, step):
    return list(range(0, n, step)) + [n]


@pytest.mark.parametrize("addr_text", [True, False])
@pytest.mark.parametrize("k", range(len(LISTS)))
def test_one_pass_equals_the_id_path(eng, k, addr_text):
    n = len(TABLE["flow_end"])
    _check(eng, TABLE, _namespaces(n, 3), _cuts(n, 2047), LISTS[k], addr_text, algo="EWMA", emit_all=True)


@pytest.mark.parametrize("host", [0, HOST])
@pytest.mark.parametrize("addr_text", [True, False])
def test_passes_and_host_store_equal_the_id_path(eng, addr_text, host):
    """A budget that takes the table to 4 passes; with a host store, the store holds exactly the kept rows."""
    n = len(BIG["flow_end"])
    st = _check(eng, BIG, _namespaces(n, 5), _cuts(n, 65536), LISTS[2], addr_text, BUDGET_4, host, rows_hint=n)
    mem = st["memory"]
    assert mem["peak_workspace_bytes"] <= BUDGET_4 and mem["passes"] >= 2
    if host:
        assert st["rounds"] == 1 and mem["stored_rows"] == st["rows_kept"] < n
    else:
        assert st["rounds"] >= 2 and mem["stored_rows"] == 0


def test_dbscan_equals_the_id_path(eng):
    t = synth.make_flows(300, 30, seed=91, dup_frac=0.2)
    n = len(t["flow_end"])
    _check(eng, t, _namespaces(n, 7), _cuts(n, 777), LISTS[2], True, algo="DBSCAN", emit_all=True)


def _small(ns_text=True, rows=1000):
    t = synth.make_flows(50, rows // 50, seed=5)
    return blocks(t, _namespaces(len(t["flow_end"]), 9), _cuts(len(t["flow_end"]), 500), ns_text, False)


def _fails(eng, job, bl):
    from theia_b200.engine import TadError
    try:
        with pytest.raises(TadError) as e:
            feed(job, bl)
        assert e.value.code == ERR_INVALID_ARG
        assert job.poll()["state"] == "FAILED"
    finally:
        job.release()
    _normal_job_ok(eng)


def test_malformed_namespace_text_fails(eng):
    """A mark that the VarUInt walk misses: found on the GPU, reported by a push or the end call."""
    bl = _small()
    data, marks = bl[1][1]["dst_ns"]
    marks = marks.copy()
    marks[3] += 1
    bl[1][1]["dst_ns"] = (data, marks)
    _fails(eng, eng.submit_stream(ns_ignore_names=LISTS[1]), bl)


def test_text_and_ids_mixed_across_blocks_fail(eng):
    bl = _small()
    bl[1] = _small(ns_text=False)[1]
    _fails(eng, eng.submit_stream(ns_ignore_names=LISTS[1]), bl)


@pytest.mark.parametrize("case", ["ids-with-text", "names-with-ids", "one-side-each"])
def test_inconsistent_lists_and_columns_fail(eng, case):
    if case == "ids-with-text":
        job, bl = eng.submit_stream(ns_ignore=[1]), _small()
    elif case == "names-with-ids":
        job, bl = eng.submit_stream(ns_ignore_names=LISTS[1]), _small(ns_text=False)
    else:
        job, bl = eng.submit_stream(ns_ignore_names=LISTS[1]), _small()
        b, txt = bl[0]
        bl[0] = (dict(b, src_ns=np.zeros(len(b["flow_end"]), dtype=np.uint32)), {"dst_ns": txt["dst_ns"]})
    _fails(eng, job, bl)


# ---- a flagged streamed job with namespace text beside an ARIMA fit ---------------------------------------------------

def _wait_fitting(job, timeout=120.0):
    t0 = time.time()
    while job.progress()["fits_done"] == 0:
        assert job.poll()["state"] in ("SCHEDULED", "RUNNING"), job.poll()
        assert time.time() - t0 < timeout, "the fit phase did not start"
        time.sleep(0.002)


@pytest.fixture(scope="module")
def long_cols():
    return _device_table([(150_000, 100, 14)])


@pytest.mark.parametrize("algo", ["EWMA", "ARIMA"])
def test_flagged_job_beside_a_fit_equals_its_solo_run(eng, long_cols, algo):
    """EWMA: runs in the yield of a tad_submit ARIMA fit.  ARIMA: fits beside it (TAD_FLAG_FIT_BESIDE).  Both with
    namespace and address text; their rows equal their solo rows."""
    t = synth.make_flows(2_000, 100, seed=21)
    bl = blocks(t, _namespaces(len(t["flow_end"]), 11), _cuts(len(t["flow_end"]), 8192), True, True)
    kw = dict(algo=algo, emit_all=True, ns_ignore_names=LISTS[2])
    solo, st_solo = _run(eng, bl, LISTS[2], True, **{k: v for k, v in kw.items() if k != "ns_ignore_names"})
    eng.set_fit_sharing(RESERVE)
    a = eng.submit(long_cols, algo="ARIMA", tad_id="A", emit_all=True)
    try:
        _wait_fitting(a)
        time.sleep(0.2)
        q = eng.submit_stream(tad_id="B", share=True, fit_beside=(algo == "ARIMA"), **kw)
        err = []
        fd = threading.Thread(target=lambda: err.append(None) if feed(q, bl) else None)
        fd.start()
        fd.join()
        st = q.wait()
        state = a.poll()["state"]
        rows = q.result()
        q.release()
        a.cancel()
    finally:
        eng.set_fit_sharing(0)
        a.wait(check=False)
        a.release()
    assert err == [None]
    assert state == "RUNNING", "B did not finish while A's fit ran"
    assert st["rows_kept"] == st_solo["rows_kept"] < st["rows_in"]
    assert_same_rows(rows, solo, what="%s with namespace text beside a fit" % algo)


# ---- the job entry point ----------------------------------------------------------------------------------------------

# (argv, environment besides TAD_STREAM_INPUT=1): connection mode with device text addresses and with push-down; the
# aggregated modes under TAD_DEVICE_TEXT=all
MODES = [([], {"TAD_DEVICE_TEXT": "1"}), ([], {"TAD_IPV4_PUSHDOWN": "1"}),
         (["--agg-flow", "external"], {"TAD_DEVICE_TEXT": "all"}), (["--agg-flow", "svc"], {"TAD_DEVICE_TEXT": "all"}),
         (["--agg-flow", "pod"], {"TAD_DEVICE_TEXT": "all"}),
         (["--agg-flow", "pod", "--pod-name", "pod-6", "--pod-namespace", "shop"], {"TAD_DEVICE_TEXT": "all"})]
ENTRY_LISTS = [["kube-system"], ["kube-system", "flow-visibility", "no-such-ns"]]


@pytest.mark.parametrize("k", range(len(ENTRY_LISTS)))
@pytest.mark.parametrize("mode", range(len(MODES)))
def test_entry_with_device_namespaces_equals_the_host_namespaces(eng, mode, k, monkeypatch):
    table = make_table(series=3000, points=100, seed=84, block_rows=65536)          # 3e5 rows
    args, env = MODES[mode]
    argv = ["--algo", "EWMA", "--id", "gpu-ns", "--ns-ignore-list", ad.json.dumps(ENTRY_LISTS[k])] + args
    for v in ("TAD_HOST_BUDGET", "TAD_DEVICE_TEXT", "TAD_IPV4_PUSHDOWN", "TAD_DEVICE_NS"):
        monkeypatch.delenv(v, raising=False)
    monkeypatch.setenv("TAD_STREAM_INPUT", "1")
    for key, v in env.items():
        monkeypatch.setenv(key, v)
    bodies = []
    for ns in ("0", "1"):
        monkeypatch.setenv("TAD_DEVICE_NS", ns)
        rec, tr = _Recording(eng), TableTransport(table, block_rows=65536)
        seen = []
        submit = rec.submit_stream
        rec.submit_stream = lambda **kw: (seen.append(sorted(kw)), submit(**kw))[1]
        assert ad.main(argv, engine=rec, transport=tr) == 0
        bodies.append(canonical_rows(tr.inserts[0][1]))
        assert ("ns_ignore_names" in seen[0]) == (ns == "1"), seen
    assert len(bodies[0]["id"]) > 1
    assert same(bodies[1], bodies[0]), (args, env, ENTRY_LISTS[k])
