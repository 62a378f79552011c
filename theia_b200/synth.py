"""Synthetic flow tables of the shapes BASELINE.json names (SURVEY.md section 8d).

Columns follow the ClickHouse ``flows`` table the reference job reads
(build/charts/theia/provisioning/datasources/create_table.sh:31-85), restricted to
what the TAD query selects (plugins/anomaly-detection/anomaly_detection.py:52-61):
sourceIP, sourceTransportPort, destinationIP, destinationTransportPort,
protocolIdentifier, flowStartSeconds, flowEndSeconds, throughput.  IPs are IPv4
packed into u32 (the host shim dictionary-encodes anything else).

``make_flows`` is the numpy generator used by tests; ``make_flows_torch`` builds
the same distribution on a torch device for the large bench configurations
(host generation of 1e8+ rows would dominate the run).
"""
from __future__ import annotations

import numpy as np

T0 = 1660199214          # 2022-08-11T06:26:54Z, the e2e fixture's flowStartSeconds
SERVICE_PORTS = np.array(
    [20, 21, 22, 23, 25, 53, 67, 68, 69, 80, 88, 110, 111, 123, 135, 137, 138, 139, 143, 161,
     179, 389, 443, 445, 465, 514, 515, 587, 636, 853, 873, 993, 995, 1080, 1194, 1433, 1521,
     1723, 1883, 2049, 2181, 2379, 2380, 3000, 3306, 3389, 4369, 5000, 5201, 5432, 5672, 5900,
     6379, 6443, 8000, 8080, 8443, 8888, 9000, 9090, 9092, 9200, 11211, 27017], dtype=np.uint16)
SPIKE_FACTORS = np.array([0.1, 2.5, 12.0])

COLUMN_DTYPES = {
    "src_ip": np.uint32, "src_port": np.uint16, "dst_ip": np.uint32, "dst_port": np.uint16,
    "proto": np.uint8, "flow_start": np.uint32, "flow_end": np.uint32, "value": np.uint64,
}


def make_flows(n_series: int, points_per_series: int, seed: int = 0, dup_frac: float = 0.0,
               shuffle: bool = True, ragged: bool = False, positive_only: bool = True) -> dict:
    """Rows = n_series * points (+ duplicates).  ``ragged`` draws per-series lengths in
    [1, 2*points) instead of a fixed length.  ``dup_frac`` re-emits that fraction of rows
    with a smaller-or-equal value (stage A's max() must collapse them)."""
    rng = np.random.default_rng(seed)
    S = n_series
    src_ip = (np.uint32(10 << 24) + rng.integers(0, 1 << 24, S, dtype=np.uint32)).astype(np.uint32)
    dst_ip = (np.uint32(10 << 24) + rng.integers(0, 1 << 24, S, dtype=np.uint32)).astype(np.uint32)
    src_port = rng.integers(1024, 65536, S).astype(np.uint16)
    dst_port = SERVICE_PORTS[rng.integers(0, len(SERVICE_PORTS), S)]
    proto = np.where(rng.random(S) < 0.8, 6, 17).astype(np.uint8)
    flow_start = (T0 + rng.integers(0, 3600, S)).astype(np.uint32)
    if ragged:
        lens = rng.integers(1, max(2, 2 * points_per_series), S)
    else:
        lens = np.full(S, points_per_series, dtype=np.int64)
    R = int(lens.sum())
    sid = np.repeat(np.arange(S), lens)
    first = np.cumsum(lens) - lens
    k = np.arange(R) - np.repeat(first, lens) + 1          # 1..n within the series
    base = np.exp(rng.uniform(np.log(1e6), np.log(1e10), S))
    val = base[sid] + rng.normal(0.0, 1.0, R) * (1e-3 * base[sid])
    spike = rng.random(R) < 0.01
    val = np.where(spike, val * SPIKE_FACTORS[rng.integers(0, 3, R)], val)
    val = np.maximum(np.rint(val), 1.0 if positive_only else 0.0).astype(np.uint64)
    cols = {
        "src_ip": src_ip[sid], "src_port": src_port[sid], "dst_ip": dst_ip[sid],
        "dst_port": dst_port[sid], "proto": proto[sid], "flow_start": flow_start[sid],
        "flow_end": (flow_start[sid].astype(np.int64) + 60 * k).astype(np.uint32),
        "value": val,
    }
    if dup_frac > 0:
        nd = int(R * dup_frac)
        pick = rng.integers(0, R, nd)
        dup = {c: v[pick].copy() for c, v in cols.items()}
        # half the duplicates carry a smaller value, half an equal one
        dup["value"] = np.where(rng.random(nd) < 0.5, dup["value"] // 2, dup["value"]).astype(np.uint64)
        cols = {c: np.concatenate([cols[c], dup[c]]) for c in cols}
    if shuffle:
        perm = rng.permutation(len(cols["value"]))
        cols = {c: v[perm] for c, v in cols.items()}
    return {c: np.ascontiguousarray(v, dtype=COLUMN_DTYPES[c]) for c, v in cols.items()}


def golden_e2e_table(values, shuffle_seed: int | None = 7, duplicates: int = 0) -> dict:
    """The single connection the reference e2e test inserts
    (test/e2e/throughputanomalydetection_test.go:401-492): 10.10.1.25:58076 ->
    10.10.1.33:5201 tcp, flowStart 2022-08-11T06:26:54Z, flowEnd = 07:26:54Z + i*60 s."""
    n = len(values)
    cols = {
        "src_ip": np.full(n, (10 << 24) | (10 << 16) | (1 << 8) | 25, dtype=np.uint32),
        "src_port": np.full(n, 58076, dtype=np.uint16),
        "dst_ip": np.full(n, (10 << 24) | (10 << 16) | (1 << 8) | 33, dtype=np.uint32),
        "dst_port": np.full(n, 5201, dtype=np.uint16),
        "proto": np.full(n, 6, dtype=np.uint8),
        "flow_start": np.full(n, T0, dtype=np.uint32),
        "flow_end": (T0 + 3600 + 60 * np.arange(n)).astype(np.uint32),
        "value": np.asarray(values, dtype=np.uint64),
    }
    if duplicates:
        cols = {c: np.concatenate([v] * (1 + duplicates)) for c, v in cols.items()}
    if shuffle_seed is not None:
        perm = np.random.default_rng(shuffle_seed).permutation(len(cols["value"]))
        cols = {c: v[perm] for c, v in cols.items()}
    return cols


def make_flows_torch(n_series: int, points_per_series: int, seed: int, device, noisy: bool = False):
    """Same distribution as ``make_flows`` (fixed length, no duplicates), generated on
    ``device`` with torch ops; returns a dict of torch tensors with the column dtypes
    widened to what torch supports (u16 -> int16 bit pattern, u32 -> int32, u64 -> int64;
    the engine reads raw bytes, so only the bit patterns matter).  ``noisy``: throughputs of a few hundred with 15 %
    noise and 4 % spikes instead of 1e6..1e10 with 0.1 % noise -- the regime in which ARIMA's Box-Cox transform is
    well conditioned (near-constant series make the reference's calculate_arima fail inside its blanket except)."""
    import torch
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    S, n = n_series, points_per_series
    R = S * n

    def ri(lo, hi, size):
        return torch.randint(lo, hi, (size,), generator=g, device=device, dtype=torch.int64)

    src_ip = (10 << 24) + ri(0, 1 << 24, S)
    dst_ip = (10 << 24) + ri(0, 1 << 24, S)
    src_port = ri(1024, 65536, S)
    ports = torch.as_tensor(SERVICE_PORTS.astype(np.int64), device=device)
    dst_port = ports[ri(0, len(SERVICE_PORTS), S)]
    proto = torch.where(torch.rand(S, generator=g, device=device) < 0.8, 6, 17)
    flow_start = T0 + ri(0, 3600, S)
    base = torch.exp(torch.empty(S, device=device, dtype=torch.float64).uniform_(
        float(np.log(1e6)), float(np.log(1e10)), generator=g))
    if noisy:
        base = torch.empty(S, device=device, dtype=torch.float64).uniform_(50.0, 500.0, generator=g)
    perm = torch.randperm(R, generator=g, device=device)         # global shuffle
    sid = perm // n
    k = perm % n + 1
    b = base[sid]
    val = b + torch.randn(R, generator=g, device=device, dtype=torch.float64) * ((0.15 if noisy else 1e-3) * b)
    spike = torch.rand(R, generator=g, device=device) < (0.04 if noisy else 0.01)
    fac = torch.as_tensor(np.array([0.5, 2.0, 3.0]) if noisy else SPIKE_FACTORS, device=device)[ri(0, 3, R)]
    val = torch.where(spike, val * fac, val)
    val = torch.clamp(torch.round(val), min=1.0).to(torch.int64)
    del b, spike, fac, perm
    cols = {
        "src_ip": src_ip[sid].to(torch.int32), "src_port": src_port[sid].to(torch.int16),
        "dst_ip": dst_ip[sid].to(torch.int32), "dst_port": dst_port[sid].to(torch.int16),
        "proto": proto[sid].to(torch.uint8), "flow_start": flow_start[sid].to(torch.int32),
        "flow_end": (flow_start[sid] + 60 * k).to(torch.int32),
        "value": val,
    }
    return cols


def make_flows_torch_sharded(series_per_gpu: int, points_per_series: int, seed: int, device, rank: int, world: int):
    """Rank `rank`'s shard of a table with world * series_per_gpu connections: global row g = sid * points + (k - 1) lives
    on rank g % world, so every rank holds exactly series_per_gpu * points rows (series_per_gpu * points is a multiple of
    world for the bench shapes; otherwise the shards differ by at most one row), every connection's points are spread over
    all ranks and NO connection is local before the exchange."""
    import torch
    g = torch.Generator(device=device)
    g.manual_seed(seed)                      # same key attributes on every rank
    S, n = series_per_gpu * world, points_per_series

    def ri(gen, lo, hi, size):
        return torch.randint(lo, hi, (size,), generator=gen, device=device, dtype=torch.int64)

    src_ip = (10 << 24) + ri(g, 0, 1 << 24, S)
    dst_ip = (10 << 24) + ri(g, 0, 1 << 24, S)
    src_port = ri(g, 1024, 65536, S)
    ports = torch.as_tensor(SERVICE_PORTS.astype(np.int64), device=device)
    dst_port = ports[ri(g, 0, len(SERVICE_PORTS), S)]
    proto = torch.where(torch.rand(S, generator=g, device=device) < 0.8, 6, 17)
    flow_start = T0 + ri(g, 0, 3600, S)
    base = torch.exp(torch.empty(S, device=device, dtype=torch.float64).uniform_(
        float(np.log(1e6)), float(np.log(1e10)), generator=g))
    g2 = torch.Generator(device=device)
    g2.manual_seed(seed * 1000 + 17 + rank)   # per-rank noise and shuffle
    total = S * n
    R = (total - rank + world - 1) // world   # global rows g = rank, rank + world, ... < total
    perm = torch.randperm(R, generator=g2, device=device)
    gl = perm * world + rank
    sid = gl // n
    k = gl % n + 1                            # 1..n
    b = base[sid]
    val = b + torch.randn(R, generator=g2, device=device, dtype=torch.float64) * (1e-3 * b)
    spike = torch.rand(R, generator=g2, device=device) < 0.01
    fac = torch.as_tensor(SPIKE_FACTORS, device=device)[ri(g2, 0, 3, R)]
    val = torch.where(spike, val * fac, val)
    val = torch.clamp(torch.round(val), min=1.0).to(torch.int64)
    del b, spike, fac, perm, gl
    return {
        "src_ip": src_ip[sid].to(torch.int32), "src_port": src_port[sid].to(torch.int16),
        "dst_ip": dst_ip[sid].to(torch.int32), "dst_port": dst_port[sid].to(torch.int16),
        "proto": proto[sid].to(torch.uint8), "flow_start": flow_start[sid].to(torch.int32),
        "flow_end": (flow_start[sid] + 60 * k).to(torch.int32),
        "value": val,
    }


def fill_columns_blocks(cols, n_series: int, points_per_series: int, seed: int, device, block_series: int = 1_000_000,
                        noisy: bool = False):
    """Fill library-owned pinned host ``Columns`` (engine.Columns, capacity >= n_series * points) block by block of
    ``block_series`` connections: each block is generated on ``device`` by ``make_flows_torch`` (seed derived from
    ``seed`` and the block index) and copied to the host, so a 1e9-row host table needs one block in HBM at a time,
    not the several-times-the-table temporaries of one ``make_flows_torch`` call.  Rows are shuffled within a block."""
    R = n_series * points_per_series
    assert cols.c.capacity >= R
    at = 0
    for b, s0 in enumerate(range(0, n_series, block_series)):
        sb = min(block_series, n_series - s0)
        t = make_flows_torch(sb, points_per_series, seed=seed * 100003 + b, device=device, noisy=noisy)
        n = sb * points_per_series
        for name, dt in COLUMN_DTYPES.items():
            cols.view(name)[at:at + n] = t[name].cpu().numpy().view(dt)
        at += n
        del t
    cols.c.rows = R
    return cols


def torch_cols_to_numpy(cols_t: dict, mask=None) -> dict:
    """Device columns (bit patterns in torch's signed dtypes) -> the numpy table the oracle takes; ``mask`` selects rows."""
    out = {}
    for name, dt in COLUMN_DTYPES.items():
        v = cols_t[name] if mask is None else cols_t[name][mask]
        out[name] = np.ascontiguousarray(v.cpu().numpy()).view(dt)
    return out
