"""Text key slots, host side: the Native reader's column span and marks (what tad_stream_push_text takes), and
tad_ch_format_names (the INSERT's String column from a dictionary and ids).  No GPU."""
import numpy as np
import pytest

from theia_b200 import clickhouse_native as cn


def string_column(values):
    """(column bytes, marks) of a Native String column of `values` (bytes), built independently of the reader."""
    enc = [cn._enc_varuint(len(v)) + v for v in values]
    starts = np.concatenate([[0], np.cumsum([len(e) for e in enc], dtype=np.uint64)])[:-1].astype(np.uint64)
    return b"".join(enc), starts[::32].copy()


def text_table(values_u32, name_of):
    """Per distinct u32 value its name (bytes) and encoded length: the text a table's address column carries."""
    uniq, inv = np.unique(values_u32, return_inverse=True)
    names = [name_of(int(v)) for v in uniq]
    return names, inv


def column_from_names(names, inv):
    """(column bytes, marks) of the rows names[inv]: the encoding joined once per distinct name, no per-row objects."""
    enc = np.empty(len(names), dtype=object)
    for i, nm in enumerate(names):
        enc[i] = cn._enc_varuint(len(nm)) + nm
    lens = np.fromiter((len(e) for e in enc), dtype=np.uint64, count=len(enc))[inv]
    starts = np.zeros(len(inv), dtype=np.uint64)
    if len(inv) > 1:
        np.cumsum(lens[:-1], out=starts[1:])
    return b"".join(enc[inv].tolist()), starts[::32].copy()


def first_appearance_ids(keys):
    """Dense ids in order of first appearance (the host Dictionary's order) and the distinct keys in that order."""
    uniq, first, inv = np.unique(keys, return_index=True, return_inverse=True)
    order = np.argsort(first, kind="stable")
    rank = np.empty(len(order), dtype=np.uint32)
    rank[order] = np.arange(len(order), dtype=np.uint32)
    return rank[inv], uniq[order]


VALUES = [b"", b"1.2.3.4", b"a" * 127, b"b" * 128, b"c" * 20000, b"\xff\xfe\x00bad", b"fd00::1", b"", b"d" * 16383,
          b"e" * 16384]


def _block(cols):
    out = [cn._enc_varuint(len(cols)), cn._enc_varuint(len(cols[0][2]))]
    for name, typ, vals in cols:
        out += [cn._enc_string(name), cn._enc_string(typ)]
        out.append(b"".join(cn._enc_varuint(len(v)) + v for v in vals) if typ == "String" else
                   np.asarray(vals, dtype=np.uint32).tobytes())
    return b"".join(out)


@pytest.mark.parametrize("rows", [1, 31, 32, 33, 100, 257])
def test_reader_span_and_marks(rows):
    rng = np.random.default_rng(rows)
    vals = [VALUES[i] for i in rng.integers(0, len(VALUES), rows)]
    other = [b"x" * int(k) for k in rng.integers(0, 200, rows)]
    body = _block([("n", "UInt32", np.arange(rows)), ("sourceIP", "String", vals), ("destinationIP", "String", other)])
    blk = next(iter(cn.read_blocks(body)))
    cols = blk[0] if isinstance(blk, tuple) else blk
    for name, want in (("sourceIP", vals), ("destinationIP", other)):
        data, marks = cols[name].text()
        exp_data, exp_marks = string_column(want)
        assert data.tobytes() == exp_data
        assert marks.dtype == np.uint64 and marks.tolist() == exp_marks.tolist()
        # the full index agrees: row 32k's payload sits after its VarUInt at the mark
        c = cols[name]
        for k, m in enumerate(marks):
            assert int(c.offsets[32 * k]) - c.start == int(m) + len(cn._enc_varuint(len(want[32 * k])))


def test_format_names_layout_and_errors():
    names = [b"", b"10.0.0.1", b"fd00::2", b"z" * 128, b"\x80\x81", b"y" * 20000]
    data = np.frombuffer(b"".join(names), dtype=np.uint8)
    offsets = np.concatenate([[0], np.cumsum([len(n) for n in names])]).astype(np.uint64)
    nm = cn.Names(data, offsets)
    ids = np.array([0, 5, 3, 3, 1, 2, 4, 0], dtype=np.uint32)
    assert cn.format_names(nm, ids) == b"".join(cn._enc_string(names[i]) for i in ids)
    assert cn.format_names(nm, np.zeros(0, dtype=np.uint32)) == b""
    with pytest.raises(ValueError):
        cn.format_names(nm, np.array([0, 6], dtype=np.uint32))
    # a short buffer through the C call
    import ctypes as C
    from theia_b200 import _lib
    out = np.empty(5, dtype=np.uint8)
    used = C.c_size_t(0)
    ids = np.array([1], dtype=np.uint32)
    assert _lib.load().tad_ch_format_names(data.ctypes.data, offsets.ctypes.data, len(names), ids.ctypes.data, 1,
                                           out.ctypes.data, out.size, C.byref(used)) == -1
    out = np.empty(9, dtype=np.uint8)
    assert _lib.load().tad_ch_format_names(data.ctypes.data, offsets.ctypes.data, len(names), ids.ctypes.data, 1,
                                           out.ctypes.data, out.size, C.byref(used)) == 0
    assert out[:used.value].tobytes() == cn._enc_string(b"10.0.0.1")


def test_tadetector_block_takes_a_device_dictionary():
    """A Names dictionary as an ip_col source writes the same bytes as the host dictionary with the same names."""
    from theia_b200 import anomaly_detection as ad
    plan = ad.plan_query()
    names = ["10.0.0.1", "fd00::1", ""]
    got = {k: np.zeros(3, dtype=np.uint32) for k in ("src_ip", "dst_ip", "flow_start", "flow_end")}
    got.update(src_ip=np.array([2, 0, 1], dtype=np.uint32), dst_ip=np.array([1, 1, 0], dtype=np.uint32),
               src_port=np.zeros(3, np.uint16), dst_port=np.zeros(3, np.uint16), proto=np.zeros(3, np.uint8),
               stddev=np.ones(3), algo_calc=np.ones(3), throughput=np.ones(3))
    host = {}
    for slot in ("src_ip", "dst_ip"):
        d = ad.Dictionary()
        d.encode(np.asarray(names, dtype=object))
        host[slot] = d
    enc = [n.encode() for n in names]
    dev = {slot: cn.Names(np.frombuffer(b"".join(enc), dtype=np.uint8),
                          np.concatenate([[0], np.cumsum([len(e) for e in enc])]).astype(np.uint64))
           for slot in ("src_ip", "dst_ip")}
    a = cn.tadetector_block_from_result(got, plan, host, "EWMA", "id")
    b = cn.tadetector_block_from_result(got, plan, dev, "EWMA", "id")
    assert a == b


def test_first_appearance_helper():
    ids, order = first_appearance_ids(np.array([7, 3, 7, 9, 3, 1], dtype=np.uint32))
    assert ids.tolist() == [0, 1, 0, 2, 1, 3] and order.tolist() == [7, 3, 9, 1]
    names, inv = text_table(np.array([5, 5, 2]), lambda v: b"n%d" % v)
    data, marks = column_from_names(names, inv)
    assert (data, marks.tolist()) == (string_column([b"n5", b"n5", b"n2"])[0], [0])


# ---- the job entry point with TAD_DEVICE_TEXT=1, on an engine double that encodes the text on the host ---------------

def _names_of(data, marks, rows):
    """The names of a text column, walked from its bytes; the walk must meet every mark, as the engine's decode checks."""
    buf = memoryview(np.asarray(data, dtype=np.uint8)).cast("B")
    p, out = 0, []
    for i in range(rows):
        if i % 32 == 0:
            assert p == int(marks[i // 32]), "a mark disagrees with the VarUInt lengths"
        n, p = cn._varuint(buf, p)
        out.append(bytes(buf[p:p + n]).decode("utf-8", "surrogateescape"))
        p += n
    assert p == len(buf)
    return out


def _text_doubles():
    from .test_job_entry_stream import StreamEngine, StreamJob

    class TextStreamJob(StreamJob):
        """Takes text slots as tad_stream_push_text does: ids in first-appearance order over the pushes, one dictionary
        per slot for the whole job (Dictionary.encode_block semantics), and names(slot) as tad_job_names gives them."""

        def __init__(self, eng, kw):
            super().__init__(eng, kw)
            from theia_b200 import anomaly_detection as ad
            self.text_dicts = {"src_ip": ad.Dictionary(), "dst_ip": ad.Dictionary()}
            self.text_slots = None

        def push(self, block, text=None):
            slots = tuple(sorted(text or ()))
            assert self.text_slots in (None, slots), "every block must make the first block's text choice"
            self.text_slots = slots
            block = dict(block)
            for slot in slots:
                assert block[slot] is None, "a text slot's u32 column is NULL"
                data, marks = text[slot]
                names = _names_of(data, marks, len(block["flow_end"]))
                block[slot] = self.text_dicts[slot].encode(np.asarray(names, dtype=object))
            self.eng.text_pushes.append(slots)
            super().push(block)

        def names(self, slot):
            enc = [n.encode("utf-8", "surrogateescape") for n in self.text_dicts[slot].names]
            offsets = np.concatenate([[0], np.cumsum([len(e) for e in enc], dtype=np.uint64)]).astype(np.uint64)
            return np.frombuffer(b"".join(enc), dtype=np.uint8), offsets

    class TextStreamEngine(StreamEngine):
        def __init__(self, rounds=1):
            super().__init__(rounds)
            self.text_pushes = []

        def submit_stream(self, **kw):
            self.jobs.append(TextStreamJob(self, kw))
            return self.jobs[-1]

    return TextStreamEngine


def _entry(monkeypatch, argv, flows, device_text, rounds=1):
    from theia_b200 import anomaly_detection as ad
    from .test_job_entry_stream import TableTransport, canonical_rows
    monkeypatch.setenv("TAD_STREAM_INPUT", "1")
    if device_text:
        monkeypatch.setenv("TAD_DEVICE_TEXT", "1")
    else:
        monkeypatch.delenv("TAD_DEVICE_TEXT", raising=False)
    eng, tr = _text_doubles()(rounds), TableTransport(flows)
    assert ad.main(argv, engine=eng, transport=tr) == 0
    (_, body), = tr.inserts
    return canonical_rows(body), eng, body


@pytest.fixture
def fixed_clock(monkeypatch):
    from theia_b200 import anomaly_detection as ad
    from .test_job_entry_stream import _FixedNow
    monkeypatch.setattr(ad, "datetime", _FixedNow)


@pytest.mark.parametrize("dual_stack", [False, True])
@pytest.mark.parametrize("rounds", [1, 2])
def test_device_text_insert_body_equals_the_host_dictionary_path(monkeypatch, fixed_clock, dual_stack, rounds):
    from .test_job_entry_stream import make_table
    flows = make_table(dual_stack=dual_stack)
    argv = ["--algo", "EWMA", "--id", "dt"]
    want, eng0, body0 = _entry(monkeypatch, argv, flows, False, rounds)
    got, eng, body = _entry(monkeypatch, argv, flows, True, rounds)
    assert len(want) > 1 and got == want and body == body0
    assert eng0.text_pushes and all(s == () for s in eng0.text_pushes)
    assert eng.text_pushes and all(s == ("dst_ip", "src_ip") for s in eng.text_pushes)


@pytest.mark.parametrize("extra", [["--agg-flow", "pod"], ["--agg-flow", "svc"], ["--agg-flow", "external"],
                                   ["--agg-flow", "pod", "--pod-label", "web", "--pod-namespace", "shop"]])
def test_other_modes_push_what_they_push_without_the_switch(monkeypatch, fixed_clock, extra):
    from .test_job_entry_stream import make_table
    flows = make_table(dual_stack=True)
    argv = ["--algo", "EWMA", "--id", "m"] + extra
    want, eng0, body0 = _entry(monkeypatch, argv, flows, False)
    got, eng, body = _entry(monkeypatch, argv, flows, True)
    assert body == body0 and all(s == () for s in eng.text_pushes)
    a, b = eng0.jobs[0].pushes, eng.jobs[0].pushes
    assert len(a) == len(b)
    for ra, rb in zip(a, b):
        assert len(ra) == len(rb)
        for pa, pb in zip(ra, rb):
            assert pa.keys() == pb.keys()
            for k in pa:
                assert (pa[k] is None and pb[k] is None) or np.array_equal(pa[k], pb[k]), k


def test_device_text_needs_no_pushdown(monkeypatch, fixed_clock):
    """With TAD_IPV4_PUSHDOWN=1 the addresses are UInt32 columns: the switch has nothing to encode."""
    from .test_job_entry_stream import make_table
    monkeypatch.setenv("TAD_IPV4_PUSHDOWN", "1")
    _, eng, _ = _entry(monkeypatch, ["--algo", "EWMA", "--id", "p"], make_table(), True)
    assert all(s == () for s in eng.text_pushes)
