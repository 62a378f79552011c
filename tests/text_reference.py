"""Plain-Python references of the device text kernels (theia_b200/csrc/tad_text.cu), and the crafted inputs of the
collision tests: the folded FNV-1a name hash, the VarUInt decode of a block's 32-row segments, a first-appearance
dictionary with the kernels' state words, and a model of the open-addressing table that counts how often a probe meets
a different name with an equal tag."""
import json
import os

import numpy as np

from theia_b200 import clickhouse_native as cn

U64 = 2 ** 64 - 1
FULL = U64
# the masks the device tests run at: the product hash; one probe chain with every tag equal; every tag equal with the
# slots spread; every name starting at slot 0 with the tags differing; 8 hash bits
MASKS = [FULL, 0, 0x00000000FFFFFFFF, 0xFFFFFFFF00000000, 0x0000000F0000000F]
# the mask-0 cases keep to this many names: every probe walks one chain
MASK0_NAMES = 16384
NS_MAX_NAMES, NS_MAX_BYTES = 1024, 32768          # kNsMaxNames, kNsMaxBytes (tad_text.h)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "text_tag_collisions.json")


def fnv_state(prefix: bytes) -> int:
    h = 1469598103934665603
    for c in prefix:
        h = ((h ^ c) * 1099511628211) & U64
    return h


def name_hash(s: bytes, mask: int = FULL) -> int:
    """name_hash of tad_text.cu: FNV-1a, folded so that the low (slot) bits see the high bytes."""
    h = fnv_state(s)
    return (h ^ (h >> 29)) & mask


def name_hashes(tails: np.ndarray, mask: int = FULL, prefix: bytes = b"") -> np.ndarray:
    """name_hash of prefix + each row of `tails` (uint8, rows x length), vectorised: uint64."""
    h = np.full(len(tails), fnv_state(prefix), dtype=np.uint64)
    for k in range(tails.shape[1]):
        h ^= tails[:, k].astype(np.uint64)
        h *= np.uint64(1099511628211)
    return (h ^ (h >> np.uint64(29))) & np.uint64(mask)


def fixture_pairs(length=None):
    """The golden pairs of distinct names sharing their hash's tag and low 12 bits, as bytes; all lengths by default."""
    with open(GOLDEN) as f:
        pairs = json.load(f)["pairs"]
    keys = [str(length)] if length is not None else sorted(pairs, key=int)
    return [(a.encode(), b.encode()) for k in keys for a, b in pairs[k]]


# ---- a Native String column cut into 32-row segments ------------------------------------------------------------------

def segments(names):
    """The encoded bytes of each 32-row segment of a String column of `names`."""
    enc = [cn._enc_varuint(len(v)) + v for v in names]
    return [b"".join(enc[k:k + 32]) for k in range(0, len(enc), 32)]


def column(segs):
    """(column bytes, marks) of a column given as its segments' bytes (each segment's first byte is its mark)."""
    marks = np.zeros(len(segs), dtype=np.uint64)
    if len(segs) > 1:
        marks[1:] = np.cumsum([len(s) for s in segs[:-1]])
    return b"".join(segs), marks


def window(data, marks, rows, lo, n):
    """The arguments of a chunk of rows [lo, lo + n) of a block of `rows` rows, as the engine stages it: the span of
    its segments' bytes, their absolute marks, the segment count and the first segment's row."""
    s0 = lo // 32
    s1 = min((rows + 31) // 32, (lo + n + 31) // 32)
    at = lambda s: int(marks[s]) if s < (rows + 31) // 32 else len(data)
    a, b = at(s0), at(s1)
    return data[a:b], marks[s0:s1].copy(), s1 - s0, s0 * 32


def decode(text, marks, nseg, seg0_row, block_rows, lo, n):
    """text_decode_kernel: (the name of each row of [lo, lo + n), error flag).  Each segment walks its rows' VarUInt
    lengths from its mark to the next mark (the span's end for the last); a segment that reads past that end, has an
    11th VarUInt byte, or does not end exactly there, gives the empty name to its rows and sets the flag."""
    span = len(text)
    out = [b""] * n
    err = False
    base = int(marks[0]) if nseg else 0
    for k in range(nseg):
        r0 = seg0_row + 32 * k
        r1 = min(r0 + 32, block_rows)
        pos = (int(marks[k]) - base) & U64
        end = (int(marks[k + 1]) - base) & U64 if k + 1 < nseg else span
        ok = pos <= end <= span
        got = {}
        r = r0
        while ok and r < r1:
            v, shift = 0, 0
            while True:
                if pos >= end or shift > 63:
                    ok = False
                    break
                b = text[pos]
                pos += 1
                v = (v | (b & 0x7F) << shift) & U64
                if not b & 0x80:
                    break
                shift += 7
            if not ok or v > end - pos:
                ok = False
                break
            got[r] = text[pos:pos + v]
            pos += v
            r += 1
        ok = ok and pos == end
        if not ok:
            err = True
        for r in range(max(r0, lo), min(r1, lo + n)):
            out[r - lo] = got[r] if ok else b""
    return out, err


# ---- the dictionary ---------------------------------------------------------------------------------------------------

class RefDict:
    """A job's text dictionary as plain Python: ids in order of first appearance, and the state words the device
    dictionary keeps (0 names, 1 arena bytes, 2 decode error, 3-4 the last chunk's new names and bytes, 5 a name missing
    from the frozen dictionary)."""

    def __init__(self):
        self.ids = {}
        self.names = []
        self.state = [0] * 6
        self.frozen = False

    def encode(self, rows, error=False):
        out = np.zeros(len(rows), dtype=np.uint32)
        new = nbytes = 0
        for i, s in enumerate(rows):
            if s not in self.ids:
                if self.frozen:
                    self.state[5] = 1
                    continue
                self.ids[s] = len(self.names)
                self.names.append(s)
                new += 1
                nbytes += len(s)
            out[i] = self.ids[s]
        self.state[0] += new
        self.state[1] += nbytes
        self.state[2] |= int(error)
        self.state[3], self.state[4] = new, nbytes
        return out


class ProbeModel:
    """The device table's probing, one row at a time (the device resolves a chunk's rows concurrently, but a slot once
    filled stays filled, so two names whose probes share a start slot and a tag meet in either order).  Counts the probes
    that compare the bytes of a different name behind an equal tag, and the longest probe."""

    def __init__(self, cap, mask):
        self.cap, self.mask = cap, mask
        self.slots = [None] * cap          # (tag, name)
        self.meetings = 0                  # probes that met a tag-equal different name
        self.longest = 0                   # slots visited by the longest probe

    def grow(self, cap):
        old = [x for x in self.slots if x is not None]
        self.cap, self.slots = cap, [None] * cap
        for tag, s in old:
            p = name_hash(s, self.mask) & (cap - 1)
            while self.slots[p] is not None:
                p = (p + 1) & (cap - 1)
            self.slots[p] = (tag, s)

    def probe(self, s):
        h = name_hash(s, self.mask)
        tag, p = h >> 32, h & (self.cap - 1)
        met, steps = False, 1
        while self.slots[p] is not None:
            t, other = self.slots[p]
            if t == tag:
                if other == s:
                    break
                met = True
            p = (p + 1) & (self.cap - 1)
            steps += 1
        else:
            self.slots[p] = (tag, s)
        self.meetings += met
        self.longest = max(self.longest, steps)


# ---- the device cases' inputs -----------------------------------------------------------------------------------------

def prefix_names():
    """Names that are prefixes of each other, the empty name, and lengths where the VarUInt prefix grows."""
    return [b"", b"a", b"aa", b"aaa", b"a" * 127, b"a" * 128, b"a" * 16383, b"a" * 16384, b"b" * 127, b"b" * 128, b"ab"]


def chunk_order_rows(pairs, first_a=True):
    """One chunk where each pair's names interleave: x x y x y y x with x the first to appear."""
    rows = []
    for a, b in pairs:
        x, y = (a, b) if first_a else (b, a)
        rows += [x, x, y, x, y, y, x]
    return rows


def random_tails(n, rng, length=12):
    return rng.integers(ord("a"), ord("z") + 1, size=(n, length), dtype=np.uint8)


def random_names(n, rng, length=12):
    return [bytes(r) for r in random_tails(n, rng, length)]


def ns_partners(mask, count, rng, length=12, prefix=b""):
    """`count` pairs (listed name, row name) of distinct prefix + random names, `length` bytes in all, with equal hashes
    under `mask`, no name in two pairs (the full hash has no such pairs: the golden pairs share 44 of its bits)."""
    bits = bin(mask).count("1")
    assert bits <= 40
    n = max(8 * count, int(np.sqrt(8.0 * count * 2.0 ** bits)) + 1)
    tails = random_tails(n, rng, length - len(prefix))
    key = name_hashes(tails, mask, prefix)
    order = np.argsort(key, kind="stable")
    ks = key[order]
    pairs, used = [], set()
    for j in np.flatnonzero(ks[1:] == ks[:-1]):
        a, b = prefix + tails[order[j]].tobytes(), prefix + tails[order[j + 1]].tobytes()
        if a != b and a not in used and b not in used:
            used.update((a, b))
            pairs.append((a, b))
            if len(pairs) == count:
                break
    assert len(pairs) == count, (mask, len(pairs))
    return pairs


def ns_case(mask, which, seed):
    """(listed names, row names): the list at kNsMaxNames names or at kNsMaxBytes bytes; under a narrowed mask every
    listed name shares its hash with an unlisted row name."""
    rng = np.random.default_rng(seed)
    if which == "names":
        count, length, prefix = NS_MAX_NAMES, 12, b""
    else:
        count, length, prefix = NS_MAX_BYTES // 128, 128, b"n" * 116
    if mask == FULL:                    # the golden pairs: equal tag and low bits, not equal hashes
        gold = [p for p in fixture_pairs() if (len(p[0]) == 128) == (length == 128)][:count]
        fill = [prefix + t.tobytes() for t in random_tails(2 * (count - len(gold)), rng, length - len(prefix))]
        pairs = gold + list(zip(fill[0::2], fill[1::2]))
    else:
        pairs = ns_partners(mask, count, rng, length, prefix)
    listed = [a for a, _ in pairs]
    assert len(listed) <= NS_MAX_NAMES and sum(len(x) for x in listed) <= NS_MAX_BYTES
    rows = listed + [b for _, b in pairs] + [x[:-1] for x in listed[:50]] + [b"", listed[0] + b"x"]
    rows = [rows[k] for k in rng.permutation(len(rows))]
    return listed, rows
