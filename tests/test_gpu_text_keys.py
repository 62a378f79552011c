"""Text key slots on the GPU (tad_stream_push_text): src_ip / dst_ip pushed as Native String column bytes give, bit for bit
and ids included, the result of the same blocks pushed with ids from a host dictionary in first-appearance order -- in one
pass, in hash-range passes over several rounds, with a host row store -- and the job's dictionary maps the ids back."""
import numpy as np
import pytest

from theia_b200 import synth
from tests.util import assert_same_rows

from .test_gpu_stream import BIG, BUDGET_4, TABLE, _normal_job_ok
from .test_text_keys import column_from_names, first_appearance_ids, text_table

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_NOMEM, ERR_STATE, ERR_CANCELLED, ERR_UNSUPPORTED = -1, -3, -5, -6, -7
HOST = 1 << 30


@pytest.fixture(scope="module")
def eng():
    """A context of its own: the budgets set here must not reach the session's engine."""
    from theia_b200.engine import TadEngine
    e = TadEngine(device=0)
    yield e
    e.close()


def name_of(v: int) -> bytes:
    """An injective text for address value v: IPv4, full and compressed IPv6, the empty name, and 128+ byte names."""
    k = v % 7
    if k == 0:
        return b"%d.%d.%d.%d" % ((v >> 24) & 255, (v >> 16) & 255, (v >> 8) & 255, v & 255)
    if k == 1:
        return b"fd00:0000:0000:0000:0000:0000:%04x:%04x" % (v >> 16, v & 0xFFFF)
    if k == 2:
        return b"fd00::%x:%x" % (v >> 16, v & 0xFFFF)
    if k == 3 and v % 49 == 3:
        return b""
    if k == 4:
        return b"host-%d." % v + b"x" * (128 + v % 300)
    return b"2001:db8::%x" % v


class TextSource:
    """One table, cut into blocks, pushed as text and as host-dictionary ids (the same rows in the same order)."""

    def __init__(self, table, cuts):
        self.t = table
        self.cuts = cuts
        self.text = {}
        self.ids = {}
        self.order = {}
        for slot in ("src_ip", "dst_ip"):
            names, inv = text_table(table[slot], name_of)
            self.text[slot] = (names, inv)
            # the empty name stands for several values: ids are over names, as the host dictionary's are
            distinct = {}
            canon = np.array([distinct.setdefault(nm, len(distinct)) for nm in names], dtype=np.int64)
            ids, order = first_appearance_ids(canon[inv])
            self.ids[slot] = ids
            listed = list(distinct)
            self.order[slot] = [listed[k] for k in order]

    def blocks(self, as_text):
        for lo, hi in zip(self.cuts[:-1], self.cuts[1:]):
            b = {k: v[lo:hi] for k, v in self.t.items()}
            if not as_text:
                b.update(src_ip=self.ids["src_ip"][lo:hi], dst_ip=self.ids["dst_ip"][lo:hi])
                yield b, None
                continue
            txt = {}
            for slot in ("src_ip", "dst_ip"):
                names, inv = self.text[slot]
                txt[slot] = column_from_names(names, inv[lo:hi])
                b[slot] = None
            yield b, txt


def run(eng, src, as_text, budget=0, host=0, **kw):
    eng.set_memory_budget(budget)
    eng.set_host_budget(host)
    job = eng.submit_stream(tad_id="text" if as_text else "ids", **kw)
    try:
        rounds, again = 0, True
        while again:
            for b, txt in src.blocks(as_text):
                job.push(b, text=txt)
            again = job.end()
            rounds += 1
        st = job.wait()
        st["rounds"] = rounds
        st["memory"] = job.memory()
        names = {s: job.names(s) for s in ("src_ip", "dst_ip")} if as_text else None
        return job.result(), st, names
    finally:
        job.release()
        eng.set_host_budget(0)


def check(eng, src, budget=0, host=0, **kw):
    ref, st_ref, _ = run(eng, src, False, budget, host, **kw)
    got, st, names = run(eng, src, True, budget, host, **kw)
    for k in ("rows_in", "rows_kept", "points", "series", "result_rows"):
        assert st[k] == st_ref[k], k
    assert_same_rows(got, ref, what="text vs host ids")
    for slot in ("src_ip", "dst_ip"):
        data, offsets = names[slot]
        got_names = [data[offsets[k]:offsets[k + 1]].tobytes() for k in range(len(offsets) - 1)]
        assert got_names == src.order[slot], slot
    return st


def odd_cuts(n, seed):
    rng = np.random.default_rng(seed)
    cuts = [0]
    sizes = [1, 31, 33, 32, 100, 2047, 4099, 65536 + 17]
    while cuts[-1] < n:
        cuts.append(min(n, cuts[-1] + int(rng.choice(sizes))))
    return cuts


@pytest.mark.parametrize("algo", ["EWMA", "DBSCAN"])
def test_parity_uneven_blocks(eng, algo):
    n = len(TABLE["flow_end"])
    st = check(eng, TextSource(TABLE, odd_cuts(n, 5)), algo=algo, emit_all=True)
    assert st["rounds"] == 1 and st["memory"]["passes"] == 1


def test_parity_arima(eng):
    t = synth.make_flows(60, 30, seed=83, dup_frac=0.1)
    check(eng, TextSource(t, odd_cuts(len(t["flow_end"]), 6)), algo="ARIMA", emit_all=True)


@pytest.mark.parametrize("host", [0, HOST])
def test_rounds_and_passes_under_a_budget(eng, host):
    n = len(BIG["flow_end"])
    src = TextSource(BIG, list(range(0, n, 65536)) + [n])
    st = check(eng, src, BUDGET_4, host, rows_hint=n)
    assert st["memory"]["passes"] >= 2
    assert st["rounds"] == 1 if host else st["rounds"] >= 2
    assert st["memory"]["peak_workspace_bytes"] <= BUDGET_4
    # the same rows in one pass
    ref, _, _ = run(eng, src, True)
    got, _, _ = run(eng, src, True, BUDGET_4, host, rows_hint=n)
    assert_same_rows(got, ref, what="passes vs one pass")


def test_store_with_uneven_blocks(eng):
    """Chunks of the store's staging start inside 32-row segments when blocks are not multiples of 32."""
    n = len(BIG["flow_end"])
    st = check(eng, TextSource(BIG, odd_cuts(n, 7)), BUDGET_4, HOST, rows_hint=n)
    assert st["rounds"] == 1 and st["memory"]["stored_rows"] > 0
    assert st["memory"]["peak_workspace_bytes"] <= BUDGET_4


def test_dictionary_takes_the_pass_columns_room(eng):
    """A dictionary that outgrows the room beside the first round's pass columns but fits by itself: that round only
    counts, the passes are planned beside the dictionary, and the rows are those of the host ids."""
    n = 200_000
    t = synth.make_flows(n, 1, seed=92)
    src = TextSource(t, list(range(0, n, 65536)) + [n])
    names = [b"%08d" % i + b"r" * 112 for i in range(n)]
    distinct = {nm: k for k, nm in enumerate(names)}
    src.text["src_ip"] = (names, np.arange(n))
    src.ids["src_ip"] = np.arange(n, dtype=np.uint32)
    src.order["src_ip"] = list(distinct)
    budget = 90 << 20
    st = check(eng, src, budget, 0)
    assert st["rounds"] >= 2 and st["memory"]["peak_workspace_bytes"] <= budget, (st["rounds"], st["memory"])


def test_cancel_while_text_chunks_run(eng):
    from theia_b200.engine import TadError
    eng.set_memory_budget(0)
    n = len(BIG["flow_end"])
    (block,) = list(TextSource(BIG, [0, n]).blocks(True))
    job = eng.submit_stream(tad_id="cancel-text")
    job.push(*block)                     # returns at once: the engine encodes and splits the block's chunks meanwhile
    job.cancel()
    with pytest.raises(TadError) as e:
        job.end()
    assert e.value.code == ERR_CANCELLED
    job.release()
    _normal_job_ok(eng)


def test_dictionary_larger_than_the_budget(eng):
    from theia_b200.engine import TadError
    n = 400_000
    t = synth.make_flows(n, 1, seed=91)
    src = TextSource(t, list(range(0, n, 65536)) + [n])
    long = {"src_ip": ([b"%08d" % i + b"q" * 300 for i in range(n)], np.arange(n)), "dst_ip": src.text["dst_ip"]}
    src.text = long
    with pytest.raises(TadError) as e:
        run(eng, src, True, 64 << 20)
    assert e.value.code == ERR_NOMEM and "dictionar" in str(e.value)
    _normal_job_ok(eng)


def test_many_names(eng):
    n = 4_000_000
    rng = np.random.default_rng(7)
    t = {"src_ip": rng.permutation(n).astype(np.uint32), "dst_ip": np.zeros(n, np.uint32),
         "src_port": np.zeros(n, np.uint16), "dst_port": np.zeros(n, np.uint16), "proto": np.full(n, 6, np.uint8),
         "flow_start": np.full(n, synth.T0, np.uint32), "flow_end": np.full(n, synth.T0 + 60, np.uint32),
         "value": rng.integers(1, 1000, n).astype(np.uint64)}
    src = TextSource(t, list(range(0, n, 1 << 20)) + [n])
    eng.set_memory_budget(0)
    job = eng.submit_stream(tad_id="many")
    try:
        for b, txt in src.blocks(True):
            job.push(b, text=txt)
        assert job.end() is False
        st = job.wait()
        data, offsets = job.names("src_ip")
    finally:
        job.release()
    want = src.order["src_ip"]
    assert st["rows_in"] == n and len(want) > 3_900_000 and len(offsets) == len(want) + 1
    assert [data[offsets[k]:offsets[k + 1]].tobytes() for k in range(len(want))] == want


def test_protocol(eng):
    import ctypes as C
    from theia_b200 import _lib as L
    from theia_b200.engine import TadError
    eng.set_memory_budget(0)
    t = synth.make_flows(100, 20, seed=88)
    src = TextSource(t, [0, 1000, 2000])
    blocks = list(src.blocks(True))
    ids = list(src.blocks(False))
    # a slot that switches between text and u32
    job = eng.submit_stream(tad_id="switch")
    job.push(*blocks[0])
    with pytest.raises(TadError) as e:
        job.push(ids[1][0])
    assert e.value.code == ERR_INVALID_ARG
    job.release()
    # names before completion
    job = eng.submit_stream(tad_id="early")
    job.push(*blocks[0])
    with pytest.raises(TadError) as e:
        job.names("src_ip")
    assert e.value.code == ERR_STATE
    job.push(*blocks[1])
    assert job.end() is False
    job.wait()
    assert len(job.names("src_ip")[1]) > 1
    job.release()
    # text on a tad_submit job
    cols = eng.columns_from_numpy(ids[0][0])
    job = eng.submit(cols)
    tx = L.TadTextColumn()
    assert eng.lib.tad_stream_push_text(job.h, C.byref(cols.c), C.byref(tx), None) == ERR_UNSUPPORTED
    job.wait()
    job.release()
    cols.free()
    # text in a device block
    from .test_gpu_stream import device_cols
    b, txt = blocks[0]
    dev = device_cols({k: v for k, v in b.items() if v is not None})
    dev.c.src_ip = dev.c.dst_ip = None
    job = eng.submit_stream(tad_id="device")
    with pytest.raises(TadError) as e:
        job.push(dev, text=txt)
    assert e.value.code == ERR_INVALID_ARG
    job.release()
    # VarUInt lengths that disagree with the marks: the job fails, the context goes on
    data, marks = txt["src_ip"]
    bad = bytearray(data)
    bad[0] = (bad[0] + 1) & 0x7F
    job = eng.submit_stream(tad_id="bad")
    with pytest.raises(TadError) as e:
        job.push(b, text={"src_ip": (bytes(bad), marks), "dst_ip": txt["dst_ip"]})
        job.end()
    assert e.value.code == ERR_INVALID_ARG
    assert job.wait(check=False)["state"] == "FAILED"
    job.release()
    _normal_job_ok(eng)


def test_cancel_mid_round(eng):
    from theia_b200.engine import TadError
    eng.set_memory_budget(0)
    t = synth.make_flows(100, 20, seed=89)
    blocks = list(TextSource(t, [0, 500, len(t["flow_end"])]).blocks(True))
    job = eng.submit_stream(tad_id="cancel")
    job.push(*blocks[0])
    job.cancel()
    with pytest.raises(TadError) as e:
        job.push(*blocks[1])
    assert e.value.code == ERR_CANCELLED
    job.release()
    _normal_job_ok(eng)
