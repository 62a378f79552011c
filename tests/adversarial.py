"""Deterministic adversarial flow tables (host only).

``synth.make_flows`` draws uniformly random keys, evenly spaced times and values between 1e6 and 1e10, so the parts of
the engine that only decide something on unusual input -- the group kernel's full-key compare and the wrap of its linear
probe, the spill sort's key heads, the exact fallback of the optimistic scatter, DBSCAN's eps ties, the strict EWMA flag,
the time sort's bins -- never meet that input.  The key hash can be inverted: ``key_hash = mix64(a ^ mix64(b + GOLD *
(proto + 1)))`` with ``mix64`` (murmur3's fmix64) a bijection and ``a = src_ip << 32 | dst_ip`` 64 free bits, so for
any ``(b, proto)`` and any target hash there is exactly one ``a``.  The generators here use that to put connections into
chosen buckets, hash tags, shared-memory start slots and pass residues, and to build distinct keys with equal 64-bit
hashes.

Every generator returns ``(table, info)``: the table in the column layout of ``synth.make_flows`` and what it is built
to reach, so a test can assert that the path was taken."""
from __future__ import annotations

import numpy as np

from theia_b200 import synth
from theia_b200.sharding import GOLD, M1, M2, key_hash, mix64

U64 = np.uint64
EPS = 250_000_000                       # DBSCAN eps (oracle/tad_oracle.py: DBSCAN_EPS)
CLASS_CAPS = (512, 768, 1024, 1280, 1536, 2048, 4096)   # group kernel capacity classes (tad_common.cuh: group_class)
SLOT_HASH_BITS = 13                     # tad_kernels.cu: kSlotHashBits
TAG_BITS = 24
_MASK64 = (1 << 64) - 1
INV_M1 = U64(pow(int(M1), -1, 1 << 64))
INV_M2 = U64(pow(int(M2), -1, 1 << 64))


# --------------------------------------------------------------------------------------------------------------------
# key crafting
# --------------------------------------------------------------------------------------------------------------------
def inv_mix64(h) -> np.ndarray:
    """Inverse of ``sharding.mix64``: an xor-shift by 33 or more bits is its own inverse, the multipliers are odd."""
    x = np.asarray(h, dtype=U64).copy()
    with np.errstate(over="ignore"):
        x ^= x >> U64(33)
        x *= INV_M2
        x ^= x >> U64(33)
        x *= INV_M1
        x ^= x >> U64(33)
    return x


def key_b(flow_start, src_port, dst_port) -> np.ndarray:
    """The second key word, as the kernels pack it: flow_start << 32 | src_port << 16 | dst_port."""
    return ((np.asarray(flow_start, dtype=U64) << U64(32)) | (np.asarray(src_port, dtype=U64) << U64(16))
            | np.asarray(dst_port, dtype=U64))


def key_for_hash(h, b, proto):
    """(src_ip, dst_ip) such that the connection (src_ip, dst_ip, b, proto) has key hash ``h``."""
    with np.errstate(over="ignore"):
        inner = mix64(np.asarray(b, dtype=U64) + GOLD * (np.asarray(proto, dtype=U64) + U64(1)))
    a = inv_mix64(h) ^ inner
    return (a >> U64(32)).astype(np.uint32), (a & U64(0xffffffff)).astype(np.uint32)


def bucket_of(h, logb: int) -> np.ndarray:
    h = np.asarray(h, dtype=U64)
    return np.zeros(h.shape, np.int64) if logb == 0 else (h >> U64(64 - logb)).astype(np.int64)


def hash_tag(h, logb: int) -> np.ndarray:
    """The 24 hash bits right below the bucket bits (tad_kernels.cu: hash_tag), which travel in the protocol word."""
    with np.errstate(over="ignore"):
        return ((np.asarray(h, dtype=U64) << U64(logb)) >> U64(40)).astype(np.int64)


def start_slot(h, logb: int, cap: int) -> np.ndarray:
    """First shared-memory hash slot the group kernel probes for a row of a ``cap``-row class:
    ``((proto_word >> 19) * HT) >> 13`` with ``proto_word = proto | tag << 8`` and ``HT = 3 * cap / 2``."""
    ht = 3 * cap // 2
    word = hash_tag(h, logb) << 8
    return ((word >> (32 - SLOT_HASH_BITS)) * ht) >> SLOT_HASH_BITS


def compose_hash(rng, n, top=None, top_bits=0, low=None, low_bits=0) -> np.ndarray:
    """n random 64-bit hashes with the top ``top_bits`` bits equal to ``top`` and the low ``low_bits`` equal to ``low``."""
    h = rng.integers(0, 1 << 63, n, dtype=np.int64).astype(U64) << U64(1)
    h |= rng.integers(0, 2, n).astype(U64)
    if top_bits:
        h &= U64(_MASK64 >> top_bits)
        h |= U64(int(top) << (64 - top_bits))
    if low_bits:
        h &= U64((_MASK64 >> low_bits) << low_bits)
        h |= U64(int(low))
    return h


def _random_b(rng, n):
    fs = (synth.T0 + rng.integers(0, 3600, n)).astype(np.uint32)
    sp = rng.integers(1024, 65536, n).astype(np.uint16)
    dp = synth.SERVICE_PORTS[rng.integers(0, len(synth.SERVICE_PORTS), n)]
    return fs, sp, dp


def keys_for_hashes(rng, hashes, proto=None):
    """One connection per target hash: random flow_start and ports, ``proto`` (default 6 or 17), solved addresses."""
    n = len(hashes)
    fs, sp, dp = _random_b(rng, n)
    pr = (np.where(rng.random(n) < 0.8, 6, 17) if proto is None else np.broadcast_to(proto, (n,))).astype(np.uint8)
    si, di = key_for_hash(hashes, key_b(fs, sp, dp), pr)
    return {"src_ip": si, "dst_ip": di, "src_port": sp, "dst_port": dp, "proto": pr, "flow_start": fs}


# --------------------------------------------------------------------------------------------------------------------
# table assembly
# --------------------------------------------------------------------------------------------------------------------
def series_rows(keys: dict, lens, times=None, values=None, rng=None, noisy=False) -> dict:
    """Rows of one series per key.  ``times`` / ``values``: per-row arrays (default: 60 s apart after flow_start, values
    like make_flows -- or, ``noisy``, a few hundred with 15 % noise, where ARIMA's Box-Cox transform is well conditioned)."""
    lens = np.asarray(lens, dtype=np.int64)
    sid = np.repeat(np.arange(len(lens)), lens)
    R = int(lens.sum())
    cols = {c: np.asarray(v)[sid] for c, v in keys.items()}
    if times is None:
        k = np.arange(R) - np.repeat(np.cumsum(lens) - lens, lens) + 1
        times = cols["flow_start"].astype(np.int64) + 60 * k
    if values is None:
        if noisy:
            base = rng.uniform(50.0, 500.0, len(lens))[sid]
            v = base * (1.0 + 0.15 * rng.normal(size=R))
        else:
            base = np.exp(rng.uniform(np.log(1e6), np.log(1e10), len(lens)))[sid]
            v = base * (1.0 + 1e-3 * rng.normal(size=R))
            v = np.where(rng.random(R) < 0.01, v * synth.SPIKE_FACTORS[rng.integers(0, 3, R)], v)
        values = np.maximum(np.rint(v), 1.0).astype(U64)
    cols["flow_end"] = np.asarray(times).astype(np.uint32)
    cols["value"] = np.asarray(values, dtype=U64)
    return cols


def concat(parts, rng=None) -> dict:
    """The parts' rows in one table, shuffled when ``rng`` is given."""
    t = {c: np.concatenate([np.asarray(p[c]) for p in parts]).astype(dt) for c, dt in synth.COLUMN_DTYPES.items()}
    if rng is not None:
        perm = rng.permutation(len(t["value"]))
        t = {c: v[perm] for c, v in t.items()}
    return {c: np.ascontiguousarray(v) for c, v in t.items()}


def n_connections(table: dict) -> int:
    key = np.stack([np.asarray(table[c]).astype(U64) for c in ("src_ip", "dst_ip", "src_port", "dst_port", "proto",
                                                                "flow_start")], 1)
    return len(np.unique(key, axis=0))


def _lens(rng, n):
    """Series lengths 1, 2, 3, 12, 40 and ragged (1..59), in turn."""
    fixed = [1, 2, 3, 12, 40, 0]
    return np.array([fixed[i % 6] or int(rng.integers(1, 60)) for i in range(n)], dtype=np.int64)


# --------------------------------------------------------------------------------------------------------------------
# generators
# --------------------------------------------------------------------------------------------------------------------
TWIN_BITS = 20      # twins share this many top hash bits: one bucket for every logB the engine picks up to 2^20 buckets


def _twin_pair(rng, protos):
    """Equal (a, b) under two protocols, searched until both hashes share their top TWIN_BITS bits."""
    p0, p1 = (U64(p) for p in protos)
    while True:
        n = 1 << 18
        a = rng.integers(0, 1 << 63, n, dtype=np.int64).astype(U64) << U64(1)
        fs, sp, dp = _random_b(rng, n)
        b = key_b(fs, sp, dp)
        with np.errstate(over="ignore"):
            h0 = mix64(a ^ mix64(b + GOLD * (p0 + U64(1))))
            h1 = mix64(a ^ mix64(b + GOLD * (p1 + U64(1))))
        hit = np.flatnonzero((h0 >> U64(64 - TWIN_BITS)) == (h1 >> U64(64 - TWIN_BITS)))
        if len(hit):
            i = hit[0]
            keys = {"src_ip": np.full(2, a[i] >> U64(32), np.uint32), "dst_ip": np.full(2, a[i] & U64(0xffffffff), np.uint32),
                    "src_port": np.full(2, sp[i]), "dst_port": np.full(2, dp[i]), "flow_start": np.full(2, fs[i]),
                    "proto": np.array([int(p0), int(p1)], np.uint8)}
            return keys, (int(h0[i]), int(h1[i]))


def collision_table(seed: int = 0, groups: int = 24, filler_series: int = 300, filler_points: int = 20,
                    twin_points: int = 2100, noisy: bool = False):
    """Groups of 2-4 distinct connections with one full 64-bit hash (differing in proto, in flow_start, in a port, or in
    all of them; the addresses differ too, solved from the hash), and protocol twins: equal addresses, ports and
    flow_start under protocols 6 / 17 and 0 / 255, whose hashes share their top TWIN_BITS bits and have no other hash of
    the table between them -- so their rows are neighbours in the spill sort.  The 6 / 17 twins carry ``twin_points``
    points each, enough to overfill their bucket in every engine.  Filler rows come from make_flows.

    info: ``groups`` (list of row-key dicts sharing one hash), ``twins`` (list of (h_lo, h_hi)), ``series``."""
    rng = np.random.default_rng(seed)
    parts, info_groups = [], []
    variants = ("proto", "flow_start", "port", "all")
    for g in range(groups):
        size = 2 + g % 3
        h = compose_hash(rng, 1)[0]
        var = variants[g % 4]
        fs, sp, dp = _random_b(rng, 1)
        fs, sp, dp = np.repeat(fs, size), np.repeat(sp, size), np.repeat(dp, size)
        pr = np.full(size, 6, np.uint8)
        if var == "proto":
            pr = np.array([6, 17, 0, 255][:size], np.uint8)
        elif var == "flow_start":
            fs = (fs + np.arange(size) * 7).astype(np.uint32)
        elif var == "port":
            if g % 8 < 4:
                sp = (sp.astype(np.int64) ^ np.arange(size)).astype(np.uint16)
            else:
                dp = (dp.astype(np.int64) + np.arange(size)).astype(np.uint16)
        else:
            fs = (fs + np.arange(size)).astype(np.uint32)
            sp = (sp.astype(np.int64) + 3 * np.arange(size)).astype(np.uint16)
            dp = (dp.astype(np.int64) ^ np.arange(size)).astype(np.uint16)
            pr = np.array([17, 6, 1, 47][:size], np.uint8)
        si, di = key_for_hash(np.full(size, h), key_b(fs, sp, dp), pr)
        keys = {"src_ip": si, "dst_ip": di, "src_port": sp, "dst_port": dp, "proto": pr, "flow_start": fs}
        info_groups.append(keys)
        parts.append(series_rows(keys, _lens(rng, size) if g % 2 else _lens(rng, size)[::-1], rng=rng, noisy=noisy))
    twins = []
    for protos, pts in (((6, 17), twin_points), ((0, 255), 12), ((17, 6), 40)):
        keys, hh = _twin_pair(rng, protos)
        twins.append(tuple(sorted(hh)))
        lens = [pts, pts + 3] if protos == (6, 17) else [pts, 1 + pts // 2]
        parts.append(series_rows(keys, lens, rng=rng, noisy=noisy))
    if filler_series:
        if noisy:
            f = series_rows(keys_for_hashes(rng, compose_hash(rng, filler_series)),
                            rng.integers(1, 2 * filler_points, filler_series), rng=rng, noisy=True)
        else:
            f = synth.make_flows(filler_series, filler_points, seed=seed + 1, ragged=True, dup_frac=0.05, shuffle=False)
        fh = key_hash(f)
        keep = np.ones(len(fh), bool)
        for lo, hi in twins:
            keep &= ~((fh > U64(lo)) & (fh < U64(hi)))
        parts.append({c: v[keep] for c, v in f.items()})
    t = concat(parts, rng)
    h = key_hash(t)
    for lo, hi in twins:        # the twins' rows are neighbours in the spill sort: no hash of the table between them
        assert not np.any((h > U64(lo)) & (h < U64(hi))), (seed, lo, hi)
    return t, {"groups": info_groups, "twins": twins, "series": n_connections(t)}


def arima_collision_table():
    """The ARIMA table of the GPU tests: 40 collision groups, the protocol twins (30 and 33 points) and 700 noisy filler
    connections of 1-29 points, about 10k rows -- enough for both buckets of a two-bucket engine to spill.  The series
    the ARIMA oracle keeps on it are committed in tests/golden/adversarial_arima_series.json."""
    return collision_table(seed=13, groups=40, filler_series=700, filler_points=15, twin_points=30, noisy=True)


def table_digest(t: dict) -> str:
    """sha256 over the table's columns, in the column order of synth.COLUMN_DTYPES."""
    import hashlib
    d = hashlib.sha256()
    for c in synth.COLUMN_DTYPES:
        d.update(np.ascontiguousarray(t[c]).tobytes())
    return d.hexdigest()


def probe_chain_table(cap: int, points: int, seed: int = 0, logb: int = 4, bucket: int = 5, same_tag_every: int = 5):
    """Bucket ``bucket`` of a ``2^logb``-bucket engine filled with exactly ``cap`` rows (``points`` per connection, the
    last connection shorter when ``cap`` is not a multiple), every connection's hash carrying the slot bits 0x1fff: the
    probe of a ``cap``-row class starts at slot HT-1 for all of them, so the chain wraps to 0 and covers ``cap`` of the
    ``HT = 3 cap / 2`` slots.  Every ``same_tag_every``-th connection shares the whole 24-bit tag (and the protocol) of
    the first one and differs only in the low hash bits: only the full-key compare tells them apart.  A few hundred
    make_flows filler rows fill the other buckets.

    info: ``bucket``, ``logb``, ``rows`` (rows in the bucket), ``series`` (connections in the bucket), ``hashes``."""
    rng = np.random.default_rng(seed * 7919 + cap * 3 + points)
    nk = -(-cap // points)
    lens = np.full(nk, points, np.int64)
    lens[-1] = cap - points * (nk - 1)
    top = (bucket << SLOT_HASH_BITS) | ((1 << SLOT_HASH_BITS) - 1)
    h = compose_hash(rng, nk, top=top, top_bits=logb + SLOT_HASH_BITS)
    tag_bits = TAG_BITS + logb
    first_top = int(h[0] >> U64(64 - tag_bits))
    same = np.arange(nk) % same_tag_every == 0
    h[same] = compose_hash(rng, int(same.sum()), top=first_top, top_bits=tag_bits)
    assert len(np.unique(h)) == nk
    pr = np.where(same, 6, np.where(rng.random(nk) < 0.7, 6, 17)).astype(np.uint8)
    keys = keys_for_hashes(rng, h, proto=pr)
    part = series_rows(keys, lens, rng=rng)
    f = synth.make_flows(150, 4, seed=seed + cap, ragged=True, shuffle=False)
    f = {c: v[bucket_of(key_hash(f), logb) != bucket] for c, v in f.items()}
    t = concat([part, f], rng)
    return t, {"bucket": bucket, "logb": logb, "rows": cap, "series": nk, "hashes": h}


def one_bucket_table(n_series: int = 300_000, points: int = 4, seed: int = 0, top_bits: int = 22):
    """``n_series`` connections of ``points`` points whose hashes share their top ``top_bits`` bits: one bucket whatever
    logB (at most 22) the engine picks.  At 1.2M rows that overfills the optimistic scatter's overflow list
    (``max(2^20, rows / 32)`` rows), so the partition falls back to the exact one and the spill path then takes one
    bucket of many series.

    info: ``rows``, ``series``, ``top`` (the shared top bits)."""
    rng = np.random.default_rng(seed)
    top = int(rng.integers(0, 1 << top_bits))
    h = compose_hash(rng, n_series, top=top, top_bits=top_bits)
    t = concat([series_rows(keys_for_hashes(rng, h), np.full(n_series, points), rng=rng)], rng)
    return t, {"rows": n_series * points, "series": n_series, "top": top, "top_bits": top_bits}


def skewed_residue_table(n_series: int = 200_000, points: int = 10, frac: float = 0.8, residue: int = 37, seed: int = 0):
    """``frac`` of the connections have hashes whose low 6 bits (the pass residue of a 64-pass split) equal ``residue``;
    the rest are uniform.  A pass plan that assumed uniform residues would put far too many rows into one pass.

    info: ``residue``, ``heavy_rows`` (rows of the heavy residue), ``rows``."""
    rng = np.random.default_rng(seed)
    heavy = rng.random(n_series) < frac
    h = compose_hash(rng, n_series)
    h[heavy] = compose_hash(rng, int(heavy.sum()), low=residue, low_bits=6)
    lens = rng.integers(1, 2 * points, n_series)
    t = concat([series_rows(keys_for_hashes(rng, h), lens, rng=rng)], rng)
    heavy_rows = int(np.sum((key_hash(t) & U64(63)) == U64(residue)))
    return t, {"residue": residue, "heavy_rows": heavy_rows, "rows": len(t["value"])}


LATTICE_LENGTHS = (4, 11, 12, 13, 100, 511, 512, 513, 767, 768, 769, 1536, 2048, 4096, 4097, 6000)
LATTICE_GAPS = (EPS - 1, EPS, EPS + 1, EPS // 2, 2 * EPS)


def _lattice_values(rng, n, base, gaps, cluster_gap):
    """Clusters of 1-5 points, ``gaps`` inside a cluster, ``cluster_gap`` (a choice) between clusters, from ``base``."""
    vals, x = [], base
    while len(vals) < n:
        size = int(rng.integers(1, 6))
        for j in range(min(size, n - len(vals))):
            if j:
                x += int(rng.choice(gaps))
            vals.append(x)
        x += int(rng.choice(cluster_gap))
    return vals


def dbscan_lattice_table(seed: int = 0, lengths=LATTICE_LENGTHS, small_n: bool = True):
    """DBSCAN's hard cases: series built from clusters of 1-5 points with gaps of eps-1, eps, eps+1, eps/2 and 2 eps
    (chains, border points, core points whose windows only partly overlap, exact eps ties), placed at about 1e9, at
    2^53 -+ k, 2^60, 2^61, 2^63 and just below 2^64 -- above 2^53 the u64 -> double rounding moves a gap to either side
    of eps.  The lengths straddle the brute-force / sweep switch (11 / 12), the capacity classes and the spill path.
    ``small_n`` adds series of 4..11 points at 1e12..1e19 with gaps eps -+ k, where the ``x^2 - 2xy + y^2`` expansion of
    sklearn's brute-force search decides the neighbourhoods.

    info: ``series``, ``values`` (one value array per connection, in time order)."""
    rng = np.random.default_rng(seed)
    bases = [10 ** 9, (1 << 53) - 7, (1 << 53) + 3, 1 << 60, 1 << 61, 1 << 63, None]
    vals = []
    for n in lengths:
        for base in bases:
            b = base if base is not None else (1 << 64) - 1 - n * 3 * EPS      # top lands within 3 eps of 2^64 - 1
            v = _lattice_values(rng, n, b, LATTICE_GAPS, (EPS + 1, EPS, 2 * EPS, 3 * EPS))
            vals.append(np.array(v, dtype=object).astype(U64))
    if small_n:
        ks = (0, 1, 1000, 10 ** 5, 10 ** 6, 10 ** 7)
        gaps = tuple(EPS + s * k for k in ks for s in (-1, 1))
        for e in range(12, 20):
            for n in range(4, 12):
                base = 10 ** e if e < 19 else 10 ** 19 - 12 * 2 * EPS
                vals.append(np.array(_lattice_values(rng, n, base, gaps, gaps), dtype=object).astype(U64))
    for v in vals:
        assert int(v.max()) <= _MASK64
    lens = np.array([len(v) for v in vals])
    keys = keys_for_hashes(rng, compose_hash(rng, len(vals)))
    series = [rng.permutation(v) for v in vals]                 # value order is not time order
    t = concat([series_rows(keys, lens, values=np.concatenate(series), rng=rng)], rng)
    return t, {"series": len(series), "values": series}


def _alone(rng, n, index_bits=5):
    """n hashes whose top ``index_bits`` bits are all different: at logB >= index_bits every connection has a bucket of
    its own."""
    assert n <= 1 << index_bits
    h = compose_hash(rng, n)
    h &= U64(_MASK64 >> index_bits)
    h |= np.arange(n).astype(U64) << U64(64 - index_bits)
    return h


EWMA_LENGTHS = (1, 2, 4095, 4096, 4097)


def ewma_edge_table(seed: int = 0, lengths=EWMA_LENGTHS):
    """Constant series (stddev 0: the strict flag compare decides every point once the EWMA has reached the value),
    all-zero series, series alternating 0 and 2^64-1, and series of 2^53 -+ 1, 2^63 and 2^64-1, each of 1, 2, 4095,
    4096 (the last count in the group kernel's reciprocal table) and 4097 (the spill path) points.  Every connection
    has a bucket of its own at logB >= 5, so the 4096-point series is scored inside the group kernel.

    info: ``series``, ``values`` (one value array per connection, in time order)."""
    rng = np.random.default_rng(seed)
    top = _MASK64
    kinds = [
        lambda n: np.full(n, 10 ** 9, U64),
        lambda n: np.full(n, (1 << 53) + 1, U64),
        lambda n: np.full(n, top, U64),
        lambda n: np.zeros(n, U64),
        lambda n: np.where(np.arange(n) % 2 == 0, U64(0), U64(top)).astype(U64),
        lambda n: np.array([(1 << 53) - 1, (1 << 53) + 1, 1 << 63, top], dtype=U64)[rng.integers(0, 4, n)],
    ]
    series = [k(n) for k in kinds for n in lengths]
    keys = keys_for_hashes(rng, _alone(rng, len(series)))
    t = concat([series_rows(keys, [len(s) for s in series], values=np.concatenate(series), rng=rng)], rng)
    return t, {"series": len(series), "values": series}


def timestamp_table(seed: int = 0, n_uniform: int = 40, n_burst: int = 16, descending: bool = True):
    """Times that break the group kernel's bin sort: series with times uniform over [0, 2^32-1] (both ends included),
    bursts of a few hundred rows within 3 s next to one far outlier (one bin holds almost the whole series), rows of
    the table in descending time order.  ``start_time`` / ``end_time`` in info equal a row's flow_start / flow_end:
    the filters keep ``flow_start == start_time`` and drop ``flow_end == end_time``."""
    rng = np.random.default_rng(seed)
    parts = []
    lens = rng.integers(5, 300, n_uniform)
    keys = keys_for_hashes(rng, compose_hash(rng, n_uniform))
    times = rng.integers(0, 1 << 32, int(lens.sum()), dtype=np.int64)
    times[0], times[1], times[-1] = 0, (1 << 32) - 1, (1 << 32) - 1
    parts.append(series_rows(keys, lens, times=times, rng=rng))
    blens = rng.integers(200, 600, n_burst)
    keys = keys_for_hashes(rng, compose_hash(rng, n_burst))
    bt = []
    for i, n in enumerate(blens):
        t0 = int(rng.integers(1, (1 << 32) - 2_000_000))
        t = t0 + rng.integers(0, 4, n)
        t[rng.integers(0, n)] = (1 << 32) - 1 if i % 2 else t0 + 1_000_000 + int(rng.integers(0, 1000))
        bt.append(t)
    parts.append(series_rows(keys, blens, times=np.concatenate(bt), rng=rng))
    t = concat(parts, None if descending else rng)
    if descending:
        order = np.argsort(-t["flow_end"].astype(np.int64), kind="stable")
        t = {c: np.ascontiguousarray(v[order]) for c, v in t.items()}
    fs = np.sort(np.unique(t["flow_start"]))
    fe = np.sort(np.unique(t["flow_end"]))
    start_time = int(fs[len(fs) // 3])
    end_time = int(fe[2 * len(fe) // 3])
    return t, {"start_time": start_time, "end_time": end_time, "series": n_uniform + n_burst}


def duplicate_table(seed: int = 0, dups: int = 4096):
    """(key, flowEndSeconds) duplicates: one series of ``dups`` copies of one point, one of 16 times x 256 copies, one of
    4097 copies (the spill path), all of values near 2^62 -- so the sum reducer wraps past 2^64, as UInt64 does -- next
    to shorter series with a few duplicates.  Every connection has a bucket of its own at logB >= 5."""
    rng = np.random.default_rng(seed)
    big = U64(1 << 62)
    lens, times, values = [], [], []

    def add(t, v):
        lens.append(len(t))
        times.append(np.asarray(t, np.int64))
        values.append(np.asarray(v, U64))

    add(np.full(dups, synth.T0 + 600), big + rng.integers(0, 1 << 40, dups).astype(U64))
    add(synth.T0 + 60 * np.repeat(np.arange(16), 256), big + rng.integers(0, 1 << 40, 4096).astype(U64))
    add(np.full(4097, synth.T0 + 120), big + rng.integers(0, 1 << 40, 4097).astype(U64))
    for n in (2, 5, 40, 300):
        add(synth.T0 + 60 * rng.integers(0, max(2, n // 3), n), rng.integers(1, 1 << 62, n).astype(U64))
    keys = keys_for_hashes(rng, _alone(rng, len(lens)))
    t = concat([series_rows(keys, lens, times=np.concatenate(times), values=np.concatenate(values), rng=rng)], rng)
    return t, {"series": len(lens)}
