"""The namespace ignore list on namespace text, host side (no GPU): the device's ignore-list test (run on the host through
tad_debug_ns_match), the header, and the job entry point under TAD_DEVICE_NS=1 on an engine double that tests the
namespace text as tad_submit_stream_filtered_ns does: no namespace column is dictionary-encoded on the host, and the
INSERT body is the host path's."""
import ctypes as C
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

from theia_b200 import _lib
from theia_b200 import anomaly_detection as ad

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMESPACES = {"default", "kube-system", "shop", "flow-visibility"}     # make_table's namespaces


def _listed(name: bytes, names, mask=~0 & (2 ** 64 - 1)) -> int:
    L = _lib.load()
    data = b"".join(names)
    off = np.zeros(len(names) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(x) for x in names])
    nb = C.create_string_buffer(name, len(name) or 1)
    db = C.create_string_buffer(data, len(data) or 1)
    return L.tad_debug_ns_match(nb, len(name), db, off.ctypes.data, len(names), mask)


LIST = [b"kube-system", b"flow-visibility", b"", b"shop", b"a" * 300]


@pytest.mark.parametrize("mask", [2 ** 64 - 1, 0, 1, 0xF])
def test_listed_is_byte_equality(mask):
    """Every mask: the full hash, and hashes narrowed so that every name (0), or many (1, 0xF), collide -- a collision
    never lists a name, since a hash match always compares the bytes."""
    for name in LIST:
        assert _listed(name, LIST, mask) == 1, name
    for name in [b"kube-syste", b"kube-system ", b"Kube-System", b"shop\x00", b"sho", b"a" * 299, b"a" * 301,
                 b"flow-visibility-x", b"\xff", "shöp".encode()]:
        assert _listed(name, LIST, mask) == 0, name
    assert _listed(b"", [b"x"], mask) == 0                   # the empty namespace is listed only when "" is
    assert _listed(b"x", [], mask) == 0 and _listed(b"", [], mask) == 0     # the empty list lists nothing


def test_random_names_against_python():
    rng = np.random.default_rng(13)
    alphabet = [b"a", b"b", b"-", b"\xc3\xa9", b"\xff", b"0"]
    pool = [b"".join(alphabet[k] for k in rng.integers(0, len(alphabet), int(rng.integers(0, 7)))) for _ in range(300)]
    for trial in range(40):
        names = [pool[k] for k in rng.integers(0, len(pool), int(rng.integers(0, 40)))]
        for mask in (2 ** 64 - 1, 3):
            for name in pool[:60]:
                assert _listed(name, names, mask) == int(name in names), (name, names, mask)


def test_names_longer_than_the_staging_per_row():
    """The text staging plans 48 bytes per row; names of any length are compared whole."""
    long = [bytes([65 + k % 26]) * n for k, n in enumerate((47, 48, 49, 64, 1000, 4096))]
    for i, name in enumerate(long):
        assert _listed(name, long) == 1
        assert _listed(name[:-1], long) == int(name[:-1] in long)
        assert _listed(name + b"A", long) == int(name + b"A" in long)
    assert _listed(b"B" * 48, long) == 1 and _listed(b"B" * 47, long) == 0


def test_header_compiles_as_c99_and_cxx17(tmp_path):
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
    src = tmp_path / "ns.c"
    src.write_text('#include "theia_tad.h"\n'
                   "int submit(tad_ctx *ctx, tad_job **out) {\n"
                   "    static const uint8_t names[] = \"kube-systemflow-visibility\";\n"
                   "    static const uint64_t offsets[] = {0, 11, 26};\n"
                   "    tad_job_spec spec = {0};\n"
                   "    tad_stream_filter_ns f = {0};\n"
                   "    f.rows.op[0] = TAD_NAME_ANY;\n"
                   "    f.rows.proto_eq = -1;\n"
                   "    f.n_ns_ignore = 2;\n"
                   "    f.ns_ignore_bytes = names;\n"
                   "    f.ns_ignore_offsets = offsets;\n"
                   "    return tad_submit_stream_filtered_ns(ctx, &spec, 0, &f, out);\n"
                   "}\n"
                   "int push(tad_job *job, const tad_columns *b, const tad_text_column *s, const tad_text_column *d) {\n"
                   "    return tad_stream_push_text_ns(job, b, NULL, NULL, s, d);\n"
                   "}\n")
    inc = os.path.join(ROOT, "include")
    subprocess.check_call([gcc, "-std=c99", "-pedantic", "-Wall", "-Werror", "-fsyntax-only", "-I", inc, "-x", "c",
                           str(src)])
    cxx = tmp_path / "ns.cc"
    cxx.write_text(src.read_text().replace("= {0}", "{}"))
    subprocess.check_call([gxx, "-std=c++17", "-Wall", "-Werror", "-fsyntax-only", "-I", inc, "-x", "c++", str(cxx)])


# ---- the job entry point with TAD_DEVICE_NS=1, on an engine double ------------------------------------------------------

def _ns_doubles():
    """The FilteredEngine double of test_text_filter, taught namespace text: a job with ``ns_ignore_names`` turns each
    block's namespace text into ids of a dictionary that starts with the list, and the CPU oracle drops the listed ids --
    what the host path pushes, so the INSERT bodies compare byte for byte."""
    from .test_text_filter import _doubles
    from .test_text_keys import _names_of
    FilteredEngine = _doubles()

    class NsEngine(FilteredEngine):
        def __init__(self, rounds=1):
            super().__init__(rounds)
            self.ns_pushes = []

        def submit_stream(self, **kw):
            names = kw.pop("ns_ignore_names", None)
            ns_dict = ad.Dictionary()
            if names is not None:
                assert list(kw["ns_ignore"]) == []
                ns_dict.encode(np.asarray([x.decode() for x in names], dtype=object))
                kw["ns_ignore"] = sorted(ns_dict.ids.values())
            job = super().submit_stream(**kw)
            job.ns_names, job.ns_dict = names, ns_dict
            push = job.push

            def push_ns(block, text=None):
                text = dict(text or {})
                block = dict(block)
                n = len(block["flow_end"])
                got = tuple(sorted(s for s in ("src_ns", "dst_ns") if s in text))
                self.ns_pushes.append(got)
                for slot in got:
                    assert job.ns_names is not None and block.get(slot) is None
                    data, marks = text.pop(slot)
                    block[slot] = job.ns_dict.encode(np.asarray(_names_of(data, marks, n), dtype=object))
                push(block, text or None)

            job.push = push_ns
            return job

    return NsEngine


@pytest.fixture
def dictionary_calls(monkeypatch):
    """The names of every String column the host dictionary-encodes (tad_ch_dictionary), one set per call."""
    L = _lib.load()
    original = L.tad_ch_dictionary
    seen = []

    def record(buf, offsets, lengths, rows, ids, first_row, n_unique):
        off = np.ctypeslib.as_array((C.c_uint64 * rows).from_address(offsets)) if rows else []
        ln = np.ctypeslib.as_array((C.c_uint32 * rows).from_address(lengths)) if rows else []
        seen.append({C.string_at(buf + int(o), int(k)).decode() for o, k in zip(off, ln)})
        return original(buf, offsets, lengths, rows, ids, first_row, n_unique)

    monkeypatch.setattr(L, "tad_ch_dictionary", record)
    return seen


def _entry(monkeypatch, argv, flows, env):
    from .test_job_entry_stream import TableTransport, canonical_rows
    for v in ("TAD_DEVICE_TEXT", "TAD_DEVICE_NS", "TAD_IPV4_PUSHDOWN"):
        monkeypatch.delenv(v, raising=False)
    monkeypatch.setenv("TAD_STREAM_INPUT", "1")
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    eng, tr = _ns_doubles()(), TableTransport(flows)
    assert ad.main(argv, engine=eng, transport=tr) == 0
    (_, body), = tr.inserts
    return canonical_rows(body), eng, body


@pytest.fixture
def fixed_clock(monkeypatch):
    from .test_job_entry_stream import _FixedNow
    monkeypatch.setattr(ad, "datetime", _FixedNow)


def _table(dual_stack=False):
    from .test_job_entry_stream import make_table
    return make_table(dual_stack=dual_stack)


# (argv, environment of the namespace-text run): connection mode with host-dictionary addresses, with device text
# addresses, with push-down addresses; the aggregated modes as TAD_DEVICE_TEXT=all takes them
CASES = {
    "connection": ([], {}),
    "connection-text": ([], {"TAD_DEVICE_TEXT": "1"}),
    "connection-pushdown": ([], {"TAD_IPV4_PUSHDOWN": "1"}),
    "external": (["--agg-flow", "external"], {"TAD_DEVICE_TEXT": "all"}),
    "svc": (["--agg-flow", "svc"], {"TAD_DEVICE_TEXT": "all"}),
    "pod": (["--agg-flow", "pod"], {"TAD_DEVICE_TEXT": "all"}),
    "pod-name-ns": (["--agg-flow", "pod", "--pod-name", "pod-6", "--pod-namespace", "shop"], {"TAD_DEVICE_TEXT": "all"}),
}
LISTS = [[], ["kube-system"], ["kube-system", "flow-visibility", "no-such-ns", ""]]


@pytest.mark.parametrize("k", range(len(LISTS)))
@pytest.mark.parametrize("case", sorted(CASES))
def test_namespace_text_writes_the_host_paths_insert_body(monkeypatch, fixed_clock, dictionary_calls, case, k):
    extra, env = CASES[case]
    flows = _table()
    argv = ["--algo", "EWMA", "--id", "ns"] + extra
    if LISTS[k]:
        argv += ["--ns-ignore-list", json.dumps(LISTS[k])]
    want, eng0, body0 = _entry(monkeypatch, argv, flows, env)
    host_calls = len(dictionary_calls)
    got, eng, body = _entry(monkeypatch, argv, flows, dict(env, TAD_DEVICE_NS="1"))
    assert len(want) > 1 and got == want and body == body0
    assert all(s == () for s in eng0.ns_pushes)
    job = eng.jobs[0]
    if LISTS[k]:
        assert eng.ns_pushes and all(s == ("dst_ns", "src_ns") for s in eng.ns_pushes)
        assert job.ns_names == [x.encode() for x in LISTS[k]] and job.kw["ns_ignore"] == list(range(len(LISTS[k])))
        # no namespace column reached the host dictionary; the host path encoded them
        assert not any(names and names <= NAMESPACES for names in dictionary_calls[host_calls:])
        assert any(names and names <= NAMESPACES for names in dictionary_calls[:host_calls])
    else:
        assert all(s == () for s in eng.ns_pushes) and job.ns_names is None


def test_two_rounds_push_the_namespace_text_again(monkeypatch, fixed_clock):
    flows = _table()
    argv = ["--algo", "EWMA", "--id", "ns2", "--ns-ignore-list", '["default"]']
    from .test_job_entry_stream import TableTransport, canonical_rows
    runs = []
    for ns in ("0", "1"):
        monkeypatch.setenv("TAD_STREAM_INPUT", "1")
        monkeypatch.setenv("TAD_DEVICE_NS", ns)
        eng, tr = _ns_doubles()(rounds=2), TableTransport(flows)
        assert ad.main(argv, engine=eng, transport=tr) == 0
        runs.append((canonical_rows(tr.inserts[0][1]), eng, tr))
    assert runs[0][0] == runs[1][0] and len(runs[1][2].selects) == 2
    eng = runs[1][1]
    assert len(eng.jobs[0].pushes) == 2 and all(s == ("dst_ns", "src_ns") for s in eng.ns_pushes)


@pytest.mark.parametrize("names", [["kube-system", "�"], ["\ud800"]])
def test_names_the_device_cannot_compare_keep_the_host_encoding(monkeypatch, fixed_clock, names):
    """The host path decodes namespaces with errors replaced (U+FFFD stands for any bytes that are not UTF-8) and a
    lone surrogate has no UTF-8 bytes: such a list keeps the host encoding."""
    flows = _table()
    argv = ["--algo", "EWMA", "--id", "nsx", "--ns-ignore-list", json.dumps(names)]
    _, eng0, body0 = _entry(monkeypatch, argv, flows, {})
    _, eng, body = _entry(monkeypatch, argv, flows, {"TAD_DEVICE_NS": "1"})
    assert body == body0 and all(s == () for s in eng.ns_pushes) and eng.jobs[0].ns_names is None


def test_a_host_masked_mode_keeps_the_host_encoding(monkeypatch, fixed_clock):
    """TAD_DEVICE_TEXT=1 keeps the pod mode's host mask: its blocks are pushed in part, so the block's namespace text
    cannot stand for them."""
    flows = _table()
    argv = ["--algo", "EWMA", "--id", "nsp", "--agg-flow", "pod", "--ns-ignore-list", '["default"]']
    _, eng0, body0 = _entry(monkeypatch, argv, flows, {"TAD_DEVICE_TEXT": "1"})
    _, eng, body = _entry(monkeypatch, argv, flows, {"TAD_DEVICE_TEXT": "1", "TAD_DEVICE_NS": "1"})
    assert body == body0 and all(s == () for s in eng.ns_pushes) and eng.jobs[0].ns_names is None


def test_submit_stream_sends_the_names_as_bytes_and_offsets(monkeypatch):
    """engine.submit_stream(ns_ignore_names=...) fills tad_stream_filter_ns: the names back to back, n + 1 offsets."""
    from theia_b200.engine import TadEngine
    seen = {}

    class Lib:
        def tad_submit_stream_filtered_ns(self, ctx, spec, hint, flt, h):
            f = flt._obj
            n = f.n_ns_ignore
            off = np.ctypeslib.as_array((C.c_uint64 * (n + 1)).from_address(f.ns_ignore_offsets)).copy()
            seen.update(n=n, off=off.tolist(), data=C.string_at(f.ns_ignore_bytes, int(off[-1])),
                        ops=list(f.rows.op), proto=f.rows.proto_eq, ids=spec._obj.n_ns_ignore)
            return 0

    eng = TadEngine.__new__(TadEngine)
    eng.lib, eng.ctx = Lib(), None
    eng.submit_stream(ns_ignore_names=[b"kube-system", b"", b"shop"])
    assert seen == {"n": 3, "off": [0, 11, 11, 15], "data": b"kube-systemshop", "ops": [0, 0], "proto": -1, "ids": 0}
