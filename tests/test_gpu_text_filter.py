"""Row predicates of a streamed job's text slots on the GPU (tad_submit_stream_filtered): the kept rows give, bit for bit after
the ids are mapped to names, the result of the same rows filtered on the host and pushed as u32 ids -- in one pass, in
hash-range passes over several rounds, and with a host row store.  Bad predicates fail with TAD_ERR_INVALID_ARG and the
context runs the next job.  The job entry point under TAD_DEVICE_TEXT=all equals the default one-shot entry in every mode."""
import numpy as np
import pytest

from theia_b200 import anomaly_detection as ad
from theia_b200 import synth
from tests.util import assert_same_rows

from .test_gpu_job_entry_stream import BLOCK, HOST, _Recording, canonical_rows, same
from .test_gpu_stream import BIG, BUDGET_4, TABLE, _normal_job_ok
from .test_gpu_text_keys import name_of
from .test_job_entry_stream import TableTransport, make_table
from .test_text_keys import column_from_names, text_table

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG = -1


@pytest.fixture(scope="module")
def eng():
    """A context of its own: the budgets set here must not reach the session's engine."""
    from theia_b200.engine import TadEngine
    e = TadEngine(device=0)
    yield e
    e.close()


def _host_keep(op, pat, names):
    if op == "eq":
        return np.array([n == pat for n in names], dtype=bool)
    if op == "nonempty":
        return np.array([len(n) > 0 for n in names], dtype=bool)
    if op == "icontains":
        p = pat.decode().lower()
        return np.array([p in n.decode("utf-8", "surrogateescape").lower() for n in names], dtype=bool)
    return np.ones(len(names), dtype=bool)


def _run(eng, table, cuts, flt, as_text, budget, host, **kw):
    """The table's rows in blocks: as text with the predicates on the GPU, or filtered here and pushed with name ids.
    Returns the result with the two address columns as canonical name ids (over both runs' names), and the status."""
    names, inv, canon = {}, {}, {}
    for slot in ("src_ip", "dst_ip"):
        names[slot], inv[slot] = text_table(table[slot], name_of)
        # the empty name stands for several values: the ids compared are over names, as the device dictionary's are
        first = {}
        canon[slot] = np.array([first.setdefault(nm, len(first)) for nm in names[slot]], dtype=np.uint32)
    keep = np.ones(len(table["flow_end"]), dtype=bool)
    if not as_text:
        for slot in ("src_ip", "dst_ip"):
            op, pat = flt.get(slot, ("any", b""))
            keep &= _host_keep(op, pat, names[slot])[inv[slot]]
        if flt.get("proto_eq", -1) >= 0:
            keep &= table["proto"] == flt["proto_eq"]
    eng.set_memory_budget(budget)
    eng.set_host_budget(host)
    job = eng.submit_stream(tad_id="f", text_filter=flt if as_text else None, **kw)
    try:
        rounds, again = 0, True
        while again:
            for lo, hi in zip(cuts[:-1], cuts[1:]):
                b = {k: v[lo:hi] for k, v in table.items()}
                if as_text:
                    txt = {slot: column_from_names(names[slot], inv[slot][lo:hi]) for slot in ("src_ip", "dst_ip")}
                    b.update(src_ip=None, dst_ip=None)
                    job.push(b, text=txt)
                else:
                    k = keep[lo:hi]
                    b = {c: v[k] for c, v in b.items()}
                    b.update(src_ip=canon["src_ip"][inv["src_ip"][lo:hi][k]], dst_ip=canon["dst_ip"][inv["dst_ip"][lo:hi][k]])
                    job.push(b)
            again = job.end()
            rounds += 1
        st = job.wait()
        st["rounds"], st["memory"] = rounds, job.memory()
        got = job.result()
        for slot in ("src_ip", "dst_ip"):
            if as_text:
                data, off = job.names(slot)
                dev = [data[off[k]:off[k + 1]].tobytes() for k in range(len(off) - 1)]
                of = {nm: int(canon[slot][i]) for i, nm in enumerate(names[slot])}
                got[slot] = np.array([of[dev[int(i)]] for i in got[slot]], dtype=np.uint32)
        return got, st
    finally:
        job.release()
        eng.set_host_budget(0)
        eng.set_memory_budget(0)


def _check(eng, table, cuts, flt, budget=0, host=0, **kw):
    ref, st_ref = _run(eng, table, cuts, flt, False, budget, host, **kw)
    got, st = _run(eng, table, cuts, flt, True, budget, host, **kw)
    for k in ("rows_kept", "points", "series", "result_rows"):
        assert st[k] == st_ref[k], (k, flt)
    assert 0 < st["rows_kept"] < len(table["flow_end"]) or not flt, flt
    assert_same_rows(got, ref, what="device predicates vs host filter %r" % (flt,))
    return st


def _filters(table):
    names = text_table(table["src_ip"], name_of)[0]
    dnames = text_table(table["dst_ip"], name_of)[0]
    some = next(n for n in names if n.startswith(b"fd00::"))
    proto = int(np.bincount(table["proto"]).argmax())
    return [
        {"src_ip": ("eq", some)},
        {"dst_ip": ("eq", dnames[len(dnames) // 2])},
        {"src_ip": ("nonempty", b"")},
        {"dst_ip": ("icontains", b"FD00::")},
        {"src_ip": ("icontains", b"HOST-"), "dst_ip": ("nonempty", b"")},
        {"proto_eq": proto},
        {"src_ip": ("icontains", b"2001:DB8"), "dst_ip": ("icontains", b":"), "proto_eq": proto},
    ]


def _cuts(n, step):
    return list(range(0, n, step)) + [n]


@pytest.mark.parametrize("k", range(7))
def test_predicates_equal_the_host_filter(eng, k):
    flt = _filters(TABLE)[k]
    _check(eng, TABLE, _cuts(len(TABLE["flow_end"]), 2047), flt, algo="EWMA", emit_all=True)


@pytest.mark.parametrize("host", [0, HOST])
@pytest.mark.parametrize("k", [2, 6])
def test_predicates_in_passes_and_with_a_host_store(eng, k, host):
    """A budget that takes the unfiltered rows to 4 passes; the kept rows run in passes of their own count."""
    n = len(BIG["flow_end"])
    st = _check(eng, BIG, _cuts(n, 65536), _filters(BIG)[k], BUDGET_4, host, rows_hint=n)
    assert st["memory"]["peak_workspace_bytes"] <= BUDGET_4
    if st["memory"]["passes"] > 1:
        assert st["rounds"] == 1 if host else st["rounds"] >= 2


def test_dbscan_with_predicates(eng):
    t = synth.make_flows(300, 30, seed=91, dup_frac=0.2)
    _check(eng, t, _cuts(len(t["flow_end"]), 777), _filters(t)[6], algo="DBSCAN", emit_all=True)


def _one_block(rows=100, text=("src_ip", "dst_ip"), proto=True):
    t = synth.make_flows(10, rows // 10, seed=5)
    b = {k: v[:rows] for k, v in t.items()}
    txt = {}
    for slot in text:
        names, inv = text_table(b[slot], name_of)
        txt[slot] = column_from_names(names, inv)
        b[slot] = None
    if not proto:
        b["proto"] = None
    return b, txt


@pytest.mark.parametrize("flt", [{"src_ip": ("bogus", b"")}, {"src_ip": (7, b"")}, {"dst_ip": ("icontains", "wéb".encode())},
                                 {"proto_eq": 256}, {"proto_eq": -2}])
def test_bad_predicates_fail_at_submit(eng, flt):
    from theia_b200.engine import TadError
    from theia_b200 import _lib as L
    if flt.get("src_ip", ("any",))[0] == "bogus":
        L.TAD_NAME_OPS["bogus"] = -1
    try:
        with pytest.raises(TadError) as e:
            eng.submit_stream(text_filter=flt)
        assert e.value.code == ERR_INVALID_ARG
    finally:
        L.TAD_NAME_OPS.pop("bogus", None)
    _normal_job_ok(eng)


def test_null_pattern_fails_at_submit(eng):
    import ctypes as C
    from theia_b200 import _lib as L
    from theia_b200.engine import TadEngine
    flt = L.TadStreamFilter()
    flt.op[0], flt.pattern_len[0], flt.proto_eq = 1, 3, -1
    spec = TadEngine._spec("EWMA", 0, 0, 0, "", False, (), 0, [])
    h = C.c_void_p()
    assert eng.lib.tad_submit_stream_filtered(eng.ctx, C.byref(spec), 0, C.byref(flt), C.byref(h)) == ERR_INVALID_ARG
    eng.lib.tad_release(h)
    _normal_job_ok(eng)


@pytest.mark.parametrize("flt,text,proto", [({"dst_ip": ("nonempty", b"")}, ("src_ip",), True),
                                            ({"proto_eq": 6}, ("src_ip",), False),
                                            ({"proto_eq": 6}, (), True)])
def test_bad_predicates_fail_at_the_first_push(eng, flt, text, proto):
    from theia_b200.engine import TadError
    b, txt = _one_block(text=text, proto=proto)
    job = eng.submit_stream(text_filter=flt)
    try:
        with pytest.raises(TadError) as e:
            job.push(b, text=txt or None)
        assert e.value.code == ERR_INVALID_ARG
    finally:
        job.release()
    _normal_job_ok(eng)


# (argv, device budget).  The svc and unfiltered pod jobs of this table hold series of 1e5+ points, more than one 1/64
# hash range may hold at 64 MiB whatever the key encoding: they take a budget that fits their largest series.
MODES = [(["--agg-flow", "external"], BUDGET_4), (["--agg-flow", "external", "--external-ip", None], BUDGET_4),
         (["--agg-flow", "svc"], 512 << 20), (["--agg-flow", "svc", "--svc-port-name", "shop/db:pg"], 512 << 20),
         (["--agg-flow", "pod"], 512 << 20), (["--agg-flow", "pod", "--pod-label", "APP", "--pod-namespace", "shop"], BUDGET_4),
         (["--agg-flow", "pod", "--pod-name", "pod-6"], BUDGET_4)]


@pytest.mark.parametrize("mode", range(len(MODES)))
def test_device_text_all_entry_equals_the_one_shot_entry(eng, mode, monkeypatch):
    table = make_table(series=20000, points=100, seed=84, dual_stack=True, block_rows=BLOCK)     # 2M rows
    d = np.asarray(table["destinationIP"])[np.asarray(table["flowType"]) == 3]
    busiest = ad.u32_to_ip(int(d[0]))
    args, small = MODES[mode]
    argv = ["--algo", "EWMA", "--id", "gpu-all"] + [busiest if a is None else a for a in args]
    for v in ("TAD_STREAM_INPUT", "TAD_HOST_BUDGET", "TAD_DEVICE_TEXT", "TAD_IPV4_PUSHDOWN"):
        monkeypatch.delenv(v, raising=False)
    eng.set_memory_budget(0)
    eng.set_host_budget(0)
    tr = TableTransport(table, block_rows=BLOCK)
    assert ad.main(argv, engine=eng, transport=tr) == 0
    want = canonical_rows(tr.inserts[0][1])
    assert len(want["id"]) > 1
    monkeypatch.setenv("TAD_STREAM_INPUT", "1")
    monkeypatch.setenv("TAD_DEVICE_TEXT", "all")
    try:
        for budget, host in ((0, None), (small, None), (small, HOST)):
            eng.set_memory_budget(budget)
            if host is None:
                monkeypatch.delenv("TAD_HOST_BUDGET", raising=False)
                eng.set_host_budget(0)
            else:
                monkeypatch.setenv("TAD_HOST_BUDGET", str(host))
            rec, tr = _Recording(eng), TableTransport(table, block_rows=BLOCK)
            assert ad.main(argv, engine=rec, transport=tr) == 0
            what = (args, budget, host)
            assert same(canonical_rows(tr.inserts[0][1]), want), what
            (mem,) = rec.memory
            # the budget forces 4 passes on the unfiltered rows; the kept rows may need fewer
            if budget:
                assert mem["peak_workspace_bytes"] <= budget, (what, mem)
            if host and mem["stored_rows"]:          # a round kept in the host store is read once
                assert len(tr.selects) == 1, (what, mem)
    finally:
        eng.set_memory_budget(0)
        eng.set_host_budget(0)
