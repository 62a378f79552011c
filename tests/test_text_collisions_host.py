"""The references and inputs of the device collision tests (test_gpu_text_collisions.py), checked without a GPU: the
Python port of the name hash against the library's, the golden pairs' collisions, the collisions each device case's
data produces under each mask, the host dictionary (tad_ch_dictionary) on colliding names, and the Python decode of a
String column's 32-row segments against the Native reader."""
import ctypes as C

import numpy as np
import pytest

from theia_b200 import _lib
from theia_b200 import clickhouse_native as cn
from tests import text_reference as R

from .test_text_keys import VALUES, _block

KEY = 0xFFFFFFFF00000FFF          # the tag and the low 12 bits
PAIRS = R.fixture_pairs()


def lib_hash(s: bytes) -> int:
    return _lib.load().tad_debug_name_hash(C.create_string_buffer(s, len(s) or 1), len(s))


def test_name_hash_port_equals_the_library():
    rng = np.random.default_rng(11)
    names = list(VALUES) + [bytes(rng.integers(0, 256, int(rng.integers(0, 64)), dtype=np.uint8)) for _ in range(200)]
    names += [bytes(rng.integers(0, 256, n, dtype=np.uint8)) for n in range(301)]
    for s in names:
        assert R.name_hash(s) == lib_hash(s), s[:20]
    tails = R.random_tails(64, rng, 20)
    want = [R.name_hash(b"pre" + t.tobytes(), 0x0F0F_FFFF_0000_FFFF) for t in tails]
    assert R.name_hashes(tails, 0x0F0F_FFFF_0000_FFFF, b"pre").tolist() == want


def test_golden_pairs_share_tag_and_low_bits():
    for length, least in ((12, 20), (127, 20), (128, 20)):
        pairs = R.fixture_pairs(length)
        assert len(pairs) >= least
        for a, b in pairs:
            assert a != b and len(a) == len(b) == length
            ha, hb = lib_hash(a), lib_hash(b)
            assert ha & KEY == hb & KEY and ha != hb, (a, b)
    names = [x for p in PAIRS for x in p]
    assert len(set(names)) == len(names)


@pytest.mark.parametrize("mask", R.MASKS, ids=["full", "0", "lo32", "hi32", "0xf0000000f"])
def test_device_cases_make_the_collisions_they_claim(mask):
    """Probing the device cases' names in order, at least one probe per golden pair meets its rival behind an equal tag
    (a pending or published entry); under mask 0 every probe walks the one chain from slot 0."""
    for first_a in (True, False):
        m = R.ProbeModel(2048, mask)
        for s in R.chunk_order_rows(PAIRS, first_a):
            m.probe(s)
        assert m.meetings >= len(PAIRS), m.meetings
    # the published case: the rivals arrive in a later chunk
    m = R.ProbeModel(2048, mask)
    for s in [a for a, _ in PAIRS] + [b for _, b in PAIRS]:
        m.probe(s)
    assert m.meetings >= len(PAIRS)
    # the rehash case: the pairs still meet after each growth
    m = R.ProbeModel(512, mask)
    for s in [a for a, _ in PAIRS]:
        m.probe(s)
    m.grow(1024)
    before = m.meetings
    for s in [b for _, b in PAIRS]:
        m.probe(s)
    assert m.meetings - before >= len(PAIRS)
    if mask == 0:                                  # one chain: every probe compares the bytes of every name before it
        assert m.longest == 2 * len(PAIRS) and m.meetings == 2 * len(PAIRS) - 1


@pytest.mark.parametrize("mask", R.MASKS[1:], ids=["0", "lo32", "hi32", "0xf0000000f"])
@pytest.mark.parametrize("which", ["names", "bytes"])
def test_namespace_cases_share_hashes(mask, which):
    listed, rows = R.ns_case(mask, which, 7)
    assert len(listed) == R.NS_MAX_NAMES if which == "names" else sum(map(len, listed)) == R.NS_MAX_BYTES
    unlisted = {R.name_hash(x, mask) for x in rows if x not in set(listed)}
    assert all(R.name_hash(x, mask) in unlisted for x in listed)


def _host_dictionary(names):
    buf = np.frombuffer(b"".join(names) or b"\0", dtype=np.uint8)
    lens = np.array([len(x) for x in names], dtype=np.uint32)
    offs = np.zeros(len(names), dtype=np.uint64)
    offs[1:] = np.cumsum(lens[:-1])
    ids, first, nu = np.zeros(len(names), np.uint32), np.zeros(len(names), np.uint64), C.c_uint32()
    assert _lib.load().tad_ch_dictionary(buf.ctypes.data, offs.ctypes.data, lens.ctypes.data, len(names),
                                         ids.ctypes.data, first.ctypes.data, C.byref(nu)) == 0
    return ids, first[:nu.value]


@pytest.mark.parametrize("seed", range(3))
def test_host_dictionary_on_colliding_names(seed):
    """tad_ch_dictionary (the host reference of the device text tests) against a Python first-appearance dictionary,
    in shuffled orders, growing from 1024 slots past 4096 (the golden pairs share a start slot up to 4096)."""
    rng = np.random.default_rng(seed)
    pool = [x for p in PAIRS for x in p] + R.prefix_names() + R.random_names(2500, rng)
    rows = [pool[k] for k in rng.integers(0, len(pool), 12000)]
    ids, first = _host_dictionary(rows)
    ref = R.RefDict()
    want = ref.encode(rows)
    assert ids.tolist() == want.tolist()
    assert [rows[r] for r in first] == ref.names and len(ref.names) > 2048


def _reader_names(names):
    body = _block([("n", "UInt32", np.arange(len(names))), ("s", "String", names)])
    blk = next(iter(cn.read_blocks(body)))
    col = (blk[0] if isinstance(blk, tuple) else blk)["s"]
    buf = np.frombuffer(col.buf, dtype=np.uint8)
    return [buf[int(o):int(o) + int(n)].tobytes() for o, n in zip(col.offsets, col.lengths)], col.text()


@pytest.mark.parametrize("rows", [1, 31, 32, 33, 100, 257])
def test_decode_reference_equals_the_native_reader(rows):
    rng = np.random.default_rng(rows)
    names = [VALUES[i] for i in rng.integers(0, len(VALUES), rows)]
    want, (data, marks) = _reader_names(names)
    data = data.tobytes()
    got, err = R.decode(data, marks, len(marks), 0, rows, 0, rows)
    assert not err and got == want == names
    # chunks that start and end inside segments, staged as the engine stages them
    for lo, n in ((0, 1), (5, 27), (31, 2), (33, rows), (rows - 1, 1)):
        n = max(0, min(n, rows - lo))
        if n == 0:
            continue
        text, mk, nseg, seg0 = R.window(data, marks, rows, lo, n)
        got, err = R.decode(text, mk, nseg, seg0, rows, lo, n)
        assert not err and got == names[lo:lo + n]


def test_decode_reference_on_malformed_segments():
    names = [b"n%03d" % k for k in range(96)]
    with pytest.raises(ValueError):                      # the reader refuses an 11th VarUInt byte too
        cn._varuint(memoryview(b"\x80" * 10 + b"\x00"), 0)
    segs = R.segments(names)
    cases = {
        "varuint-11": b"\x80" * 10 + b"\x00",
        "varuint-10-past": b"\xff" * 9 + b"\x01",
        "length-past-end": cn._enc_varuint(len(segs[1]) + 5),
    }
    for kind, head in cases.items():
        bad = list(segs)
        bad[1] = head + segs[1]
        data, marks = R.column(bad)
        got, err = R.decode(data, marks, 3, 0, 96, 0, 96)
        assert err and got == names[:32] + [b""] * 32 + names[64:], kind
    # rows that end short of the next mark; a mark past the span
    bad = list(segs)
    bad[1] = segs[1] + b"zz"
    data, marks = R.column(bad)
    got, err = R.decode(data, marks, 3, 0, 96, 0, 96)
    assert err and got == names[:32] + [b""] * 32 + names[64:]
    data, marks = R.column(segs)
    marks[2] = len(data) + 1
    got, err = R.decode(data, marks, 3, 0, 96, 0, 96)
    assert err and got == names[:32] + [b""] * 64
