"""Regenerate text_tag_collisions.json: pairs of distinct names whose folded FNV-1a hashes (the text dictionaries' and
the ignore list's name_hash) agree in the high 32 bits (the slot tag) and in the low 12 bits (the first slot of every
table of up to 4096 slots).  Two such names meet in one probe chain with equal tags, so the dictionary's byte
comparison alone tells them apart.

Candidates are random lower-case letters (sequential names such as counters spread their hashes too evenly to collide
in 44 bits at this count).  The 127- and 128-byte pairs share a fixed prefix: the search starts from the FNV state after
it, so only the random tail is hashed.  A shared suffix would not keep a collision: the names agree in 44 bits of the
folded hash, not in the 64-bit FNV state.

    python tests/golden/make_text_collisions.py        # under a minute and about 2 GB of memory on one CPU core
"""
import json
import os

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "text_tag_collisions.json")
BASIS, PRIME = np.uint64(1469598103934665603), np.uint64(1099511628211)
KEY_MASK = np.uint64(0xFFFFFFFF00000FFF)        # tag and the low 12 bits
SEED, LOG2_CANDIDATES, TAIL = 20260501, 25, 12
# (name length, prefix): the prefix fills the name up to a random tail of TAIL letters
SEARCHES = [(12, b""), (127, b"p" * (127 - TAIL)), (128, b"q" * (128 - TAIL))]


def fnv_state(prefix: bytes) -> int:
    h = 1469598103934665603
    for c in prefix:
        h = ((h ^ c) * 1099511628211) & (2 ** 64 - 1)
    return h


def fold(h):
    """The fold that makes the low (slot) bits see the high bytes."""
    return h ^ (h >> np.uint64(29))


def name_hashes(tails: np.ndarray, state: int) -> np.ndarray:
    """name_hash of prefix + tail for every row of `tails` (uint8, rows x TAIL), from the FNV state after the prefix."""
    h = np.full(len(tails), state, dtype=np.uint64)
    for k in range(tails.shape[1]):
        h ^= tails[:, k].astype(np.uint64)
        h *= PRIME
    return fold(h)


def search(prefix: bytes, rng: np.random.Generator, log2_n: int):
    """Distinct prefix + tail names in pairs whose hashes share KEY_MASK's bits."""
    tails = rng.integers(ord("a"), ord("z") + 1, size=(1 << log2_n, TAIL), dtype=np.uint8)
    key = name_hashes(tails, fnv_state(prefix)) & KEY_MASK
    order = np.argsort(key, kind="stable")
    ks = key[order]
    same = np.flatnonzero(ks[1:] == ks[:-1])
    pairs = []
    for j in same:
        a, b = prefix + tails[order[j]].tobytes(), prefix + tails[order[j + 1]].tobytes()
        if a != b:
            pairs.append(sorted([a.decode(), b.decode()]))
    return sorted(pairs)


def main():
    rng = np.random.default_rng(SEED)
    out = {"candidates_per_length": 1 << LOG2_CANDIDATES, "seed": SEED, "key_mask": "0x%016x" % int(KEY_MASK),
           "pairs": {}}
    for length, prefix in SEARCHES:
        assert len(prefix) + TAIL == length
        out["pairs"][str(length)] = search(prefix, rng, LOG2_CANDIDATES)
        print("%d-byte names: %d pairs from %d candidates" % (length, len(out["pairs"][str(length)]),
                                                              1 << LOG2_CANDIDATES))
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
