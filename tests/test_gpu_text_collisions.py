"""The device text dictionary and the namespace ignore list on names whose hashes collide, kernel by kernel against plain
Python (tests/text_reference.py).  Collisions come from the golden pairs (distinct names sharing the hash's tag and low
12 bits, so they meet in one probe chain with equal tags under the product hash) and from hash masks that make every
tag equal (0, 0xFFFFFFFF), every start slot equal (0, 0xFFFFFFFF00000000) or both often (0x0000000F0000000F).  Every
encode checks the ids, the names in id order with their stored hashes, and state words 0-5.  Then engines under
TAD_DEBUG_TEXT_MASK give the host-id path's rows bit for bit, and a later round that brings a new name fails the job."""
import ctypes as C

import numpy as np
import pytest

from theia_b200 import _lib
from theia_b200 import clickhouse_native as cn
from tests import text_reference as R

from . import test_gpu_ns_text as nt
from . import test_gpu_text_keys as tk
from .test_gpu_group_detect import make_engine
from .test_gpu_stream import BIG, BUDGET_4, TABLE, _normal_job_ok
from .test_text_keys import column_from_names

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG = -1
MASK_IDS = ["full", "0", "lo32", "hi32", "0xf0000000f"]


def _buf(b: bytes):
    return np.frombuffer(b or b"\0", dtype=np.uint8)


class DevDict:
    """The device dictionary harness (tad_debug_text_dict_*)."""

    def __init__(self, cap, mask):
        self.L = _lib.load()
        self.h = C.c_void_p()
        assert self.L.tad_debug_text_dict_new(0, cap, mask, C.byref(self.h)) == 0

    def encode(self, text, marks, nseg, seg0, rows, lo, n):
        ids, st = np.zeros(max(n, 1), dtype=np.uint32), np.zeros(8, dtype=np.uint64)
        tb, mk = _buf(text), np.ascontiguousarray(marks, dtype=np.uint64)
        rc = self.L.tad_debug_text_dict_encode(self.h, tb.ctypes.data, len(text), mk.ctypes.data if len(mk) else None,
                                               nseg, seg0, rows, lo, n, ids.ctypes.data, st.ctypes.data)
        return rc, ids[:n], st

    def names(self):
        names, nbytes = C.c_uint64(), C.c_uint64()
        assert self.L.tad_debug_text_dict_names(self.h, C.byref(names), C.byref(nbytes), None, None, None) == 0
        arena = np.zeros(max(nbytes.value, 1), dtype=np.uint8)
        off = np.zeros(names.value + 1, dtype=np.uint64)
        hashes = np.zeros(max(names.value, 1), dtype=np.uint64)
        assert self.L.tad_debug_text_dict_names(self.h, C.byref(names), C.byref(nbytes), arena.ctypes.data,
                                                off.ctypes.data, hashes.ctypes.data) == 0
        a = arena.tobytes()
        return [a[off[k]:off[k + 1]] for k in range(names.value)], hashes[:names.value].tolist()

    def close(self):
        assert self.L.tad_debug_text_dict_free(self.h) == 0


class Both:
    """A device dictionary and its Python reference, fed the same chunks."""

    def __init__(self, cap, mask):
        self.mask = mask
        self.dev = DevDict(cap, mask)
        self.ref = R.RefDict()

    def chunk(self, data, marks, rows, lo, n):
        text, mk, nseg, seg0 = R.window(data, marks, rows, lo, n)
        rc, ids, st = self.dev.encode(text, mk, nseg, seg0, rows, lo, n)
        assert rc == 0
        names, err = R.decode(text, mk, nseg, seg0, rows, lo, n)
        want = self.ref.encode(names, err)
        assert st[:6].tolist() == self.ref.state, (st[:6].tolist(), self.ref.state)
        bad = np.flatnonzero(ids != want)
        assert not len(bad), [(int(i), names[i][:20], int(ids[i]), int(want[i])) for i in bad[:5]]
        got, hashes = self.dev.names()
        assert got == self.ref.names
        assert hashes == [R.name_hash(s, self.mask) for s in got]
        return ids

    def block(self, names, cuts=None):
        """`names` as one block, encoded in one chunk or in chunks [cuts[k], cuts[k + 1])."""
        data, marks = R.column(R.segments(names))
        cuts = cuts or [0, len(names)]
        for lo, hi in zip(cuts[:-1], cuts[1:]):
            self.chunk(data, marks, len(names), lo, hi - lo)

    def close(self):
        self.dev.close()


@pytest.fixture
def both():
    made = []

    def make(cap, mask):
        made.append(Both(cap, mask))
        return made[-1]

    yield make
    for b in made:
        b.close()


PAIRS = R.fixture_pairs()
mask_param = pytest.mark.parametrize("mask", R.MASKS, ids=MASK_IDS)


@mask_param
@pytest.mark.parametrize("first_a", [True, False])
def test_order_inside_one_chunk(both, mask, first_a):
    """Each pair's names interleave in one chunk: a name's later rows come before and after its rival's first row."""
    both(2048, mask).block(R.chunk_order_rows(PAIRS, first_a))


@mask_param
def test_a_tag_equal_name_already_in_the_dictionary(both, mask):
    """The second chunk's rows meet their rival published by the first chunk (the arena comparison), not pending."""
    d = both(2048, mask)
    d.block([a for a, _ in PAIRS] * 2)
    d.block([x for a, b in PAIRS for x in (b, a, b)])
    rng = np.random.default_rng(1)
    rows = [x for p in PAIRS for x in p]
    d.block([rows[k] for k in rng.permutation(len(rows))])


@mask_param
def test_prefixes_and_the_empty_name(both, mask):
    d = both(1024, mask)
    names = R.prefix_names()
    rng = np.random.default_rng(2)
    d.block([names[k] for k in rng.integers(0, len(names), 200)])
    d.block(names[::-1] + [x for p in PAIRS[:20] for x in p] + names)


@mask_param
def test_awkward_chunk_windows(both, mask):
    """Chunks that start and end inside 32-row segments, and chunks of 1 and 31 rows, over one block."""
    rng = np.random.default_rng(3)
    pool = [x for p in PAIRS for x in p] + R.prefix_names()[:6]
    rows = [pool[k] for k in rng.integers(0, len(pool), 400)]
    cuts, sizes = [0], [1, 31, 5, 33, 64, 17, 1, 31, 100, 7]
    while cuts[-1] < len(rows):
        cuts.append(min(len(rows), cuts[-1] + sizes[len(cuts) % len(sizes)]))
    both(2048, mask).block(rows, cuts)


@mask_param
def test_rehash(both, mask):
    """The table grows between chunks (cleared, every name re-inserted from its stored hash); the ids stay those of one
    table, and colliding names met after each growth still resolve."""
    rng = np.random.default_rng(4)
    d = both(512, mask)
    filler = R.random_names(900, rng)
    d.block([a for a, _ in PAIRS] + filler[:100])
    assert d.dev.L.tad_debug_text_dict_grow(d.dev.h, 256) == ERR_INVALID_ARG       # 200 names do not fit half of 256
    assert d.dev.L.tad_debug_text_dict_grow(d.dev.h, 1000) == ERR_INVALID_ARG      # not a power of two
    assert d.dev.L.tad_debug_text_dict_grow(d.dev.h, 1024) == 0
    d.block([x for a, b in PAIRS for x in (b, a)] + filler[100:200])
    assert d.dev.L.tad_debug_text_dict_grow(d.dev.h, 4096) == 0
    rows = [x for p in PAIRS for x in p] + filler
    d.block([rows[k] for k in rng.permutation(len(rows))])
    assert d.dev.L.tad_debug_text_dict_grow(d.dev.h, 8192) == 0
    d.block(rows[::-1])


@mask_param
def test_load_at_the_limit(both, mask):
    """Chunks at exactly 2 * (names + n) == cap; one row more is refused before any kernel runs."""
    rng = np.random.default_rng(5)
    d = both(1024, mask)
    first = [x for p in PAIRS[:75] for x in p]
    d.block(first * 2)                                     # 150 names
    rest = [b for _, b in PAIRS[75:]] + R.random_names(400, rng)
    n = 512 - 150
    data, marks = R.column(R.segments(rest[:n + 1]))
    text, mk, nseg, seg0 = R.window(data, marks, n + 1, 0, n + 1)
    rc, _, st = d.dev.encode(text, mk, nseg, seg0, n + 1, 0, n + 1)
    assert rc == ERR_INVALID_ARG and d.dev.names()[0] == d.ref.names
    d.block(rest[:n])
    assert d.ref.state[0] == 512


@mask_param
def test_frozen_dictionary(both, mask):
    """After the freeze, the names it holds resolve (colliders included); a tag-equal name it lacks sets state[5] and
    gets id 0, and no name is added."""
    d = both(1024, mask)
    held = [a for a, _ in PAIRS] + R.prefix_names()
    d.block(held)
    assert d.dev.L.tad_debug_text_dict_freeze(d.dev.h) == 0
    d.ref.frozen = True
    d.block(held[::-1])
    assert d.ref.state[5] == 0
    rows = [x for a, b in PAIRS for x in (a, b)]
    data, marks = R.column(R.segments(rows))
    ids = d.chunk(data, marks, len(rows), 0, len(rows))
    assert d.ref.state[5] == 1 and not ids[1::2].any() and ids[0::2].tolist() == list(range(len(PAIRS)))


def _malformed(kind, names):
    """(column bytes, marks, failing segments) of a 160-row block whose segment 2 (or, for mark-past-span, 3 and 4) is
    corrupt."""
    segs = R.segments(names)
    bad = {2}
    if kind == "varuint-11":                   # an 11th VarUInt byte: the shift > 63 guard
        segs[2] = b"\x80" * 10 + b"\x00" + segs[2]
    elif kind == "varuint-10-past":            # a 10-byte VarUInt whose value runs past the segment
        segs[2] = b"\xff" * 9 + b"\x01" + segs[2]
    elif kind == "length-past-end":
        segs[2] = cn._enc_varuint(len(segs[2]) + 5) + segs[2]
    elif kind == "short-of-mark":              # the rows end before the next mark
        segs[2] = segs[2] + b"zz"
    data, marks = R.column(segs)
    if kind == "mark-past-span":
        marks[4] = len(data) + 7
        bad = {3, 4}
    return data, marks, bad


@mask_param
@pytest.mark.parametrize("kind", ["varuint-11", "varuint-10-past", "length-past-end", "short-of-mark", "mark-past-span"])
def test_malformed_columns(both, mask, kind):
    """The failing segments' rows, and only theirs, encode as the empty name; state[2] is set."""
    rng = np.random.default_rng(6)
    pool = [x for p in PAIRS[:40] for x in p if len(x) < 100] + [b"x", b"xy"]
    names = [pool[k] for k in rng.integers(0, len(pool), 160)]
    data, marks, bad = _malformed(kind, names)
    got, err = R.decode(data, marks, 5, 0, 160, 0, 160)
    assert err
    for r in range(160):
        assert got[r] == (b"" if r // 32 in bad else names[r]), r
    d = both(1024, mask)
    d.chunk(data, marks, 160, 0, 160)
    assert d.ref.state[2] == 1
    d.chunk(data, marks, 160, 45, 70)                      # a window that starts in segment 1 and ends in segment 3


# ---- the namespace ignore list -----------------------------------------------------------------------------------------

def _ns_device(listed, mask, names, lo, n):
    L = _lib.load()
    lb = _buf(b"".join(listed))
    off = np.zeros(len(listed) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(x) for x in listed])
    data, marks = R.column(R.segments(names))
    text, mk, nseg, seg0 = R.window(data, marks, len(names), lo, n)
    tb = _buf(text)
    verdict, err = np.zeros(max(n, 1), dtype=np.uint32), C.c_uint64(0)
    assert L.tad_debug_ns_match_device(0, lb.ctypes.data, off.ctypes.data, len(listed), mask, tb.ctypes.data,
                                       len(text), mk.ctypes.data, nseg, seg0, len(names), lo, n, verdict.ctypes.data,
                                       C.byref(err)) == 0
    return verdict[:n], err.value


@mask_param
@pytest.mark.parametrize("which", ["names", "bytes"])
def test_namespace_lookup(mask, which):
    """launch_ns_match against set membership and against its host twin tad_debug_ns_match, image and lookup under the
    same mask."""
    from .test_ns_text import _listed
    listed, rows = R.ns_case(mask, which, 7)
    want = np.array([x in set(listed) for x in rows], dtype=np.uint32)
    if mask != R.FULL:
        hashes = {R.name_hash(x, mask) for x in rows if x not in set(listed)}
        assert all(R.name_hash(x, mask) in hashes for x in listed)
    for lo, n in ((0, len(rows)), (45, len(rows) - 90)):
        verdict, err = _ns_device(listed, mask, rows, lo, n)
        assert err == 0
        assert verdict.tolist() == want[lo:lo + n].tolist()
    for x in rows[:40]:
        assert _listed(x, listed, mask) == int(x in set(listed))


def test_harness_refuses_what_the_kernels_cannot_take():
    """A capacity that is not a power of two, rows outside the staged segments."""
    L = _lib.load()
    h = C.c_void_p()
    assert L.tad_debug_text_dict_new(0, 1000, R.FULL, C.byref(h)) == ERR_INVALID_ARG
    d = DevDict(64, R.FULL)
    try:
        data, marks = R.column(R.segments([b"a"] * 40))
        rc, _, _ = d.encode(data, marks, 1, 0, 40, 0, 33)       # row 32 is in a segment not staged
        assert rc == ERR_INVALID_ARG
        rc, _, _ = d.encode(data, marks, 2, 0, 40, 0, 33)       # 2 * 33 > 64
        assert rc == ERR_INVALID_ARG
        rc, ids, st = d.encode(data, marks, 2, 0, 40, 0, 32)
        assert rc == 0 and st[0] == 1 and not ids.any()
    finally:
        d.close()


# ---- engines under TAD_DEBUG_TEXT_MASK ---------------------------------------------------------------------------------

@pytest.fixture(scope="module", params=["0x000FFFFF000FFFFF", "0x000000FF000000FF"], ids=["wide", "narrow"])
def masked(request):
    eng = make_engine(TAD_DEBUG_TEXT_MASK=request.param)
    eng.text_mask = int(request.param, 16)
    yield eng
    eng.close()


def test_masked_uneven_blocks(masked):
    n = len(TABLE["flow_end"])
    st = tk.check(masked, tk.TextSource(TABLE, tk.odd_cuts(n, 5)), algo="EWMA", emit_all=True)
    assert st["rounds"] == 1


@pytest.mark.parametrize("host", [0, tk.HOST])
def test_masked_rounds_and_passes(masked, host):
    tk.test_rounds_and_passes_under_a_budget(masked, host)


def test_masked_dictionary_takes_the_pass_columns_room(masked):
    tk.test_dictionary_takes_the_pass_columns_room(masked)


def test_masked_namespace_list(masked):
    n = len(TABLE["flow_end"])
    nt._check(masked, TABLE, nt._namespaces(n, 3), nt._cuts(n, 2047), nt.LISTS[2], True, algo="EWMA", emit_all=True)


def _absent_name(existing: bytes, mask: int) -> bytes:
    """A name that is not `existing` but, under a narrow mask, hashes as it does (so its probe meets it)."""
    if bin(mask).count("1") > 24:
        return b"absent-" + existing
    rng = np.random.default_rng(8)
    tails = R.random_tails(1 << 22, rng)
    hit = np.flatnonzero(R.name_hashes(tails, mask) == np.uint64(R.name_hash(existing, mask)))
    assert len(hit)
    return tails[hit[0]].tobytes()


def test_a_later_round_brings_a_name_the_first_did_not(masked):
    """Under a budget without a host store every round reads the source again; a name in round 2 that round 1 did not
    bring fails the job (the frozen dictionary cannot give it an id), and the context runs the next job."""
    from theia_b200.engine import TadError
    n = len(BIG["flow_end"])
    src = tk.TextSource(BIG, list(range(0, n, 65536)) + [n])
    names, inv = src.text["src_ip"]
    new = _absent_name(names[int(inv[0])], masked.text_mask)
    assert new not in set(names)
    masked.set_memory_budget(BUDGET_4)
    masked.set_host_budget(0)
    job = masked.submit_stream(tad_id="changed", rows_hint=n)
    rounds = 0
    try:
        with pytest.raises(TadError) as e:
            again = True
            while again:
                for k, (b, txt) in enumerate(src.blocks(True)):
                    if rounds and k == 0:
                        changed = inv[:len(b["flow_end"])].copy()
                        changed[7] = len(names)
                        txt["src_ip"] = column_from_names(names + [new], changed)
                    job.push(b, text=txt)
                again = job.end()
                rounds += 1
        assert e.value.code == ERR_INVALID_ARG and "source changed between reads" in str(e.value), str(e.value)
        assert rounds == 1
    finally:
        job.release()
        masked.set_memory_budget(0)
    _normal_job_ok(masked)
