"""Row predicates of a streamed job's text slots, host side (no GPU): the device's name predicate (run on the host through
tad_debug_name_match) against Python's own string semantics, and the job entry point under TAD_DEVICE_TEXT=all on an engine
double that evaluates the predicates as tad_submit_stream_filtered does."""
import ctypes as C
import json
import time

import numpy as np
import pytest

from theia_b200 import _lib
from theia_b200 import anomaly_detection as ad

EQ, NONEMPTY, ICONTAINS = 1, 2, 3
ALPHABET = ["a", "A", "i", "I", "k", "K", "b", "x", "-", "%", "_", " ", "0", "İ", "K", "ı", "é", "ß",
            "Σ", "̇", "\U0001f600", "Ā", "ↄ"]
PAT_ALPHABET = ["a", "A", "i", "I", "k", "K", "b", "x", "-", "%", "_", " ", "0"]


def _match(op, name: bytes, pat: bytes) -> int:
    L = _lib.load()
    nb = C.create_string_buffer(name, len(name) or 1)
    pb = C.create_string_buffer(pat, len(pat) or 1)
    return L.tad_debug_name_match(op, nb, len(name), pb, len(pat))


def _names(rng, count):
    out = []
    for _ in range(count):
        n = int(rng.integers(0, 9))
        out.append("".join(ALPHABET[k] for k in rng.integers(0, len(ALPHABET), n)))
    return out


def test_icontains_equals_python_lower_in_lower():
    rng = np.random.default_rng(7)
    names = _names(rng, 600) + ["", "İ", "İX", "xİ", "K", "KI", "KelvinK", "ab", "AB"]
    pats = ["", "i", "k", "I", "K", "ik", "ki", "i̇"[:1], "ab", "aB", "xi", "kk", "%_", "a" * 10]
    pats += ["".join(PAT_ALPHABET[k] for k in rng.integers(0, len(PAT_ALPHABET), int(rng.integers(1, 4))))
             for _ in range(60)]
    checked = hits = 0
    for name in names:
        # patterns taken from the name itself: at its ends, in the middle, and longer than the name
        ascii_part = "".join(ch for ch in name.lower() if ch.isascii())
        own = [ascii_part[:2], ascii_part[-2:], ascii_part, ascii_part + "z"]
        for pat in pats + own:
            want = pat.lower() in name.lower()
            got = _match(ICONTAINS, name.encode(), pat.encode())
            assert got == int(want), (name, pat)
            checked += 1
            hits += want
    assert checked > 40000 and hits > 1000
    # the two non-ASCII code points that lower-case to ASCII, and their neighbours that do not
    assert _match(ICONTAINS, "İ".encode(), b"i") == 1
    assert _match(ICONTAINS, "İb".encode(), b"ib") == 0            # U+0130 -> i U+0307: the dot comes between
    assert _match(ICONTAINS, "aKb".encode(), b"AKB") == 1
    assert _match(ICONTAINS, "ı".encode(), b"i") == 0              # dotless i stays non-ASCII


def test_eq_and_nonempty_compare_bytes():
    rng = np.random.default_rng(3)
    names = _names(rng, 300) + [""]
    for name in names:
        b = name.encode()
        assert _match(NONEMPTY, b, b"") == int(len(b) > 0)
        assert _match(EQ, b, b) == 1
        assert _match(EQ, b, b.upper()) == int(b == b.upper())
        assert _match(EQ, b, b + b"x") == 0
        assert _match(EQ, b, b[:-1]) == int(len(b) == 0)
    assert _match(EQ, b"\xff\xfe", b"\xff\xfe") == 1
    assert _match(0, b"anything", b"") == 1
    assert _match(4, b"a", b"a") == -1


# ---- the job entry point with TAD_DEVICE_TEXT=all, on an engine double ------------------------------------------------

def _doubles():
    from .test_job_entry_stream import StreamEngine, StreamJob
    from .test_text_keys import _names_of

    def keep_of(op, pattern, names):
        if op == "eq":
            return np.array([n.encode("utf-8", "surrogateescape") == pattern for n in names], dtype=bool)
        if op == "nonempty":
            return np.array([len(n) > 0 for n in names], dtype=bool)
        if op == "icontains":
            p = pattern.decode().lower()
            return np.array([p in n.lower() for n in names], dtype=bool)
        return np.ones(len(names), dtype=bool)

    class FilteredJob(StreamJob):
        """tad_submit_stream_filtered as the engine runs it: every pushed row's text names enter the slot's dictionary
        (ids in first-appearance order over all pushed rows), then the rows whose predicates fail are dropped.  The result
        order of the GPU engine is its own; this double orders it as the host path's oracle does, by the ids the host
        dictionary gives (Dictionary.encode_block: block by block, the names the kept rows use, in their first appearance
        over the block's rows), so that the INSERT bodies can be compared byte for byte."""

        def __init__(self, eng, kw):
            super().__init__(eng, kw)
            self.flt = kw.pop("text_filter", None)
            self.dicts = {"src_ip": ad.Dictionary(), "dst_ip": ad.Dictionary()}
            self.text_slots = None
            self.pushed_rows = [0]
            self.rank = {"src_ip": {}, "dst_ip": {}}           # device id -> host dictionary id

        def push(self, block, text=None):
            slots = tuple(sorted(text or ()))
            assert self.text_slots in (None, slots), "every block must make the first block's text choice"
            self.text_slots = slots
            block = dict(block)
            n = len(block["flow_end"])
            keep = np.ones(n, dtype=bool)
            flt = self.flt or {}
            for slot in slots:
                assert block[slot] is None
                data, marks = text[slot]
                names = _names_of(data, marks, n)
                block[slot] = self.dicts[slot].encode(np.asarray(names, dtype=object))
                op, pat = flt.get(slot, ("any", b""))
                keep &= keep_of(op, pat, names)
            for slot in ("src_ip", "dst_ip"):
                assert flt.get(slot, ("any",))[0] == "any" or slot in slots
            if flt.get("proto_eq", -1) >= 0:
                assert slots and block["proto"] is not None
                keep &= np.asarray(block["proto"]) == flt["proto_eq"]
            if self.rounds == 0:
                for slot in slots:
                    ids = block[slot]
                    _, at = np.unique(ids, return_index=True)
                    rank = self.rank[slot]
                    for d in ids[np.sort(at)]:                    # first appearance over the block's rows
                        if int(d) not in rank and keep[ids == d].any():
                            rank[int(d)] = len(rank)
            self.pushed_rows[-1] += n
            self.eng.text_pushes.append(slots)
            super().push({k: (None if v is None else np.asarray(v)[keep]) for k, v in block.items()})

        def end(self):
            again = super().end()
            if again:
                self.pushed_rows.append(0)
            return again

        def wait(self):
            first = self.pushes[0]
            back = {}
            for slot in self.text_slots or ():
                order = np.zeros(len(self.rank[slot]), dtype=np.uint32)
                rank = np.zeros(len(self.dicts[slot].names) + 1, dtype=np.uint32)
                for d, r in self.rank[slot].items():
                    order[r], rank[d] = d, r
                for p in first:
                    p[slot] = rank[p[slot]]
                back[slot] = order
            st = super().wait()
            for slot, order in back.items():
                self.got[slot] = order[np.asarray(self.got[slot], dtype=np.int64)].astype(np.uint32)
            return st

        def names(self, slot):
            enc = [n.encode("utf-8", "surrogateescape") for n in self.dicts[slot].names]
            offsets = np.concatenate([[0], np.cumsum([len(e) for e in enc], dtype=np.uint64)]).astype(np.uint64)
            return np.frombuffer(b"".join(enc), dtype=np.uint8), offsets

    class FilteredEngine(StreamEngine):
        def __init__(self, rounds=1):
            super().__init__(rounds)
            self.text_pushes = []

        def submit_stream(self, **kw):
            self.jobs.append(FilteredJob(self, kw))
            return self.jobs[-1]

    return FilteredEngine


def _entry(monkeypatch, argv, flows, device_text, rounds=1):
    from .test_job_entry_stream import TableTransport, canonical_rows
    monkeypatch.setenv("TAD_STREAM_INPUT", "1")
    if device_text:
        monkeypatch.setenv("TAD_DEVICE_TEXT", device_text)
    else:
        monkeypatch.delenv("TAD_DEVICE_TEXT", raising=False)
    eng, tr = _doubles()(rounds), TableTransport(flows)
    assert ad.main(argv, engine=eng, transport=tr) == 0
    (_, body), = tr.inserts
    return canonical_rows(body), eng, body


@pytest.fixture
def fixed_clock(monkeypatch):
    from .test_job_entry_stream import _FixedNow
    monkeypatch.setattr(ad, "datetime", _FixedNow)


def _table(dual_stack):
    from .test_job_entry_stream import make_table
    return make_table(dual_stack=dual_stack)


def _busiest_external_ip(flows):
    d = np.asarray(flows["destinationIP"])[np.asarray(flows["flowType"]) == 3]
    v, c = np.unique(d, return_counts=True)
    return ad.u32_to_ip(int(v[np.argmax(c)]))


MODES = {
    "connection": [],
    "external": ["--agg-flow", "external"],
    "external-ip": ["--agg-flow", "external", "--external-ip", None],
    "svc": ["--agg-flow", "svc"],
    "svc-name": ["--agg-flow", "svc", "--svc-port-name", "shop/db:pg"],
    "pod": ["--agg-flow", "pod"],
    "pod-label": ["--agg-flow", "pod", "--pod-label", "WEB"],
    "pod-label-ns": ["--agg-flow", "pod", "--pod-label", "app", "--pod-namespace", "shop"],
    "pod-name": ["--agg-flow", "pod", "--pod-name", "pod-6"],
    "pod-name-ns": ["--agg-flow", "pod", "--pod-name", "pod-6", "--pod-namespace", "shop"],
}
TEXT_SLOTS = {"connection": ("dst_ip", "src_ip"), "external": ("dst_ip",), "svc": ("src_ip",), "pod": ("dst_ip", "src_ip")}


@pytest.mark.parametrize("dual_stack", [False, True])
@pytest.mark.parametrize("rounds", [1, 2])
@pytest.mark.parametrize("ns", [False, True])
@pytest.mark.parametrize("mode", sorted(MODES))
def test_device_predicates_write_the_host_paths_insert_body(monkeypatch, fixed_clock, mode, ns, rounds, dual_stack):
    flows = _table(dual_stack)
    argv = ["--algo", "EWMA", "--id", "f"] + [_busiest_external_ip(flows) if a is None else a for a in MODES[mode]]
    if ns:
        argv += ["--ns-ignore-list", json.dumps(["kube-system"])]
    want, eng0, body0 = _entry(monkeypatch, argv, flows, None, rounds)
    got, eng, body = _entry(monkeypatch, argv, flows, "all", rounds)
    assert len(want) > 1 and got == want and body == body0
    assert all(s == () for s in eng0.text_pushes)
    assert eng.text_pushes and all(s == TEXT_SLOTS[mode.split("-")[0]] for s in eng.text_pushes)
    # every row of every block is pushed, once per branch and round
    job = eng.jobs[0]
    branches = 2 if mode.startswith("pod") else 1
    assert job.pushed_rows == [len(flows["flowEndSeconds"]) * branches] * rounds


def test_non_ascii_pod_label_keeps_the_host_encoding(monkeypatch, fixed_clock):
    from .test_job_entry_stream import make_table
    flows = make_table()
    argv = ["--algo", "EWMA", "--id", "u", "--agg-flow", "pod", "--pod-label", "wéb"]
    _, eng0, body0 = _entry(monkeypatch, argv, flows, None)
    _, eng, body = _entry(monkeypatch, argv, flows, "all")
    assert body == body0 and all(s == () for s in eng.text_pushes)
    assert eng.jobs[0].flt is None
    _same_pushes(eng0.jobs[0].pushes, eng.jobs[0].pushes)


def _same_pushes(a, b):
    assert len(a) == len(b)
    for ra, rb in zip(a, b):
        assert len(ra) == len(rb)
        for pa, pb in zip(ra, rb):
            assert pa.keys() == pb.keys()
            for k in pa:
                assert (pa[k] is None and pb[k] is None) or np.array_equal(pa[k], pb[k]), k


@pytest.mark.parametrize("mode", ["external", "svc"])
def test_blocks_with_a_non_key_start_bound_keep_the_host_encoding(mode):
    """run_engine_stream over blocks that carry flowStartSeconds where it is not a key: its lower bound is a host
    predicate, so the mode pushes exactly what it pushes without device text."""
    from theia_b200 import clickhouse_native as chn
    from .test_job_entry_stream import TYPES, make_table
    flows = make_table()
    t0 = int(np.median(np.asarray(flows["flowStartSeconds"])))
    start = time.strftime("%Y-%m-%d %H:%M:%S", time.gmtime(t0))
    cols = ["flowStartSeconds", "flowEndSeconds", "throughput", "destinationIP", "flowType", "destinationServicePortName"]

    def blocks():
        n = len(flows["flowEndSeconds"])
        for lo in range(0, n, 4000):
            spec = [(c, TYPES.get(c, "String"), np.asarray(flows[c])[lo:lo + 4000]) for c in cols]
            for blk, _types, _rows in chn.read_blocks(chn.write_native(spec)):
                yield blk

    runs = []
    for device_text in (False, "all"):
        eng = _doubles()()
        ad.run_engine_stream(eng, "EWMA", blocks, start_time=start, agg_flow=mode, device_text=device_text)
        runs.append(eng)
    assert runs[1].jobs[0].flt is None and all(s == () for s in runs[1].text_pushes)
    _same_pushes(runs[0].jobs[0].pushes, runs[1].jobs[0].pushes)
