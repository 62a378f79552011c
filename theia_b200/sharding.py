"""Host-side mirror of how the engine shards a job across the GPUs of one box (DESIGN.md section 6).

Rows arrive range-sharded by row index; the owner of a connection is chosen by the top bits of the
same 64-bit key hash the kernels use (theia_b200/csrc/tad_common.cuh: key_hash), so after one
all-to-all every series is local to exactly one rank.  These helpers let the host (and the tests)
predict ownership without a GPU."""
from __future__ import annotations

import numpy as np

M1 = np.uint64(0xff51afd7ed558ccd)
M2 = np.uint64(0xc4ceb9fe1a85ec53)
GOLD = np.uint64(0x9e3779b97f4a7c15)
GROUP_TARGET = 768


def mix64(x: np.ndarray) -> np.ndarray:
    x = x.astype(np.uint64)
    with np.errstate(over="ignore"):
        x = x ^ (x >> np.uint64(33))
        x = x * M1
        x = x ^ (x >> np.uint64(33))
        x = x * M2
        x = x ^ (x >> np.uint64(33))
    return x


def key_hash(table: dict) -> np.ndarray:
    n = len(table["flow_end"])

    def col(name):
        a = table.get(name)
        return np.zeros(n, dtype=np.uint64) if a is None else np.asarray(a).astype(np.uint64)

    a = (col("src_ip") << np.uint64(32)) | col("dst_ip")
    b = (col("flow_start") << np.uint64(32)) | (col("src_port") << np.uint64(16)) | col("dst_port")
    with np.errstate(over="ignore"):
        return mix64(a ^ mix64(b + GOLD * (col("proto") + np.uint64(1))))


def pick_logb(total_rows: int, world: int = 1) -> int:
    target = GROUP_TARGET * (2 if world >= 4 else 1)      # tad_engine.cu: pick_logb
    logb = 0
    while logb < 22 and (total_rows >> logb) > target:
        logb += 1
    logw = max(0, (world - 1).bit_length())
    return max(logb, logw)


def owner_rank(table: dict, world: int, total_rows: int | None = None) -> np.ndarray:
    """Rank that owns each row's connection."""
    if world == 1:
        return np.zeros(len(table["flow_end"]), dtype=np.int64)
    total = len(table["flow_end"]) if total_rows is None else total_rows
    logb = pick_logb(total, world)
    logw = (world - 1).bit_length()
    bucket = key_hash(table) >> np.uint64(64 - logb)
    return (bucket >> np.uint64(logb - logw)).astype(np.int64)


def pass_of(table: dict, passes: int) -> np.ndarray:
    """Hash-range pass of each row when a single-GPU job runs in ``passes`` passes (a power of two up to 64): the LOW
    key-hash bits (tad_kernels.cu: pass_split_kernel), disjoint from the bucket / owner-rank bits at the top."""
    assert passes >= 1 and passes & (passes - 1) == 0 and passes <= 64
    return (key_hash(table) & np.uint64(passes - 1)).astype(np.int64)


def shard_rows(table: dict, rank: int, world: int) -> dict:
    """Range-shard by row index (how north_star hands rows to the GPUs)."""
    n = len(table["flow_end"])
    lo, hi = n * rank // world, n * (rank + 1) // world
    return {k: (None if v is None else v[lo:hi]) for k, v in table.items()}
