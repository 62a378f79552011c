"""Column-wise restatement of the C oracle (oracle/tad_oracle.c) for EWMA and DBSCAN.  TEST INFRASTRUCTURE ONLY.

The C oracle runs one series at a time, which takes minutes on a 10^8-row table.  Both detectors can be computed over
all series at once instead, with the same IEEE FP64 operations in the same order, so that a whole full-size table can
be checked in seconds:

* stage A  rows sorted by the full key (src_ip, src_port, dst_ip, dst_port, proto, flow_start) and flow_end -- never by
  the key hash, which the engine has to tell colliding keys apart under -- then duplicates of (key, flow_end) reduced
  with ``np.maximum.reduceat`` or a u64 ``np.add.reduceat`` that wraps mod 2^64 like UInt64.
* stage B  Welford's update (Spark's CentralMomentAgg) as one numpy operation per step i over every series that has an
  i-th point: with the series ordered longest first those are a prefix.  The division by the running count is
  correctly rounded in numpy as in the kernels (tad_kernels.cu: kRcpTable), so the bits agree.
* stage C  EWMA in the same steps; the flag is the strict ``|x - e| > stddev``, never true for a one-point series
  (NaN stddev).  DBSCAN (1-D, eps 2.5e8, 4 samples) from each point's neighbourhood:
  - n >= 12: within a value-sorted series the neighbourhood ``fl(|xi - xj|) <= eps`` is a contiguous window, because
    rounding is monotone.  A point is core iff it has a left points and 3 - a right points in its window for some a;
    it is noise iff it is not core and neither its nearest core to the left nor to the right lies in its window.
  - n <= 11: sklearn's brute-force expansion ``fl(fl(xi xi - 2 xi xj) + xj xj)`` against eps^2, over an 11 x 11 block
    per series.
* output  the rows of ``tad_oracle.canonicalize`` order: key columns, then flow_end.

``run_job`` takes the arguments of ``c_oracle.run_job`` and returns what it returns, in canonical order.  The row sorts
(by key, and DBSCAN's by series and value) are numpy's unless ``sort_device`` names a torch device: only the order
comes from there, and both orders are checked on the host; the arithmetic is numpy FP64 on the host either way.
``max_chunk_rows`` splits a larger table by source address into pieces computed separately, ``workers`` at a time,
which bounds the working set next to a table of 10^9 rows.
"""
from __future__ import annotations

import numpy as np

from oracle.tad_oracle import DBSCAN_EPS, DBSCAN_MIN_SAMPLES, OUT_COLUMNS, _out_dtype

ALGO_EWMA, ALGO_DBSCAN = 0, 2
REDUCE_MAX, REDUCE_SUM = 0, 1
BRUTE_MAX_N = 11        # sklearn searches by brute force up to 11 points (tad_oracle.calculate_dbscan_anomaly)
U64 = np.uint64
_SIGN = U64(1 << 63)
_COLS = {"src_ip": np.uint32, "src_port": np.uint16, "dst_ip": np.uint32, "dst_port": np.uint16, "proto": np.uint8,
         "flow_start": np.uint32, "flow_end": np.uint32, "value": np.uint64}


# --------------------------------------------------------------------------------------------------------------------
# stage A
# --------------------------------------------------------------------------------------------------------------------
def _key_words(t):
    """The canonical order (src_ip, src_port, dst_ip, dst_port, proto, flow_start, flow_end) as three u64 words compared
    most significant first: 32 + 16 + 16 | 16 + 16 + 8 + 24 | 8 + 32 bits."""
    def u(name, shift=0, mask=None):
        w = t[name].astype(U64)
        if mask is not None:
            w &= U64(mask)
        if shift > 0:
            w <<= U64(shift)
        elif shift < 0:
            w >>= U64(-shift)
        return w

    w0 = u("src_ip", 32)
    w0 |= u("src_port", 16)
    w0 |= u("dst_ip", -16)
    w1 = u("dst_ip", 48, 0xffff)
    w1 |= u("dst_port", 32)
    w1 |= u("proto", 24)
    w1 |= u("flow_start", -8)
    w2 = u("flow_start", 32, 0xff)
    w2 |= u("flow_end")
    return w0, w1, w2


def _argsort_lex(words, sort_device=None):
    """Order of the rows by the u64 words, the first most significant (stable)."""
    if sort_device is None:
        return np.lexsort(tuple(reversed(words)))
    import torch
    order = None
    for w in reversed(words):                              # least significant first, each sort stable
        k = torch.from_numpy((w ^ _SIGN).view(np.int64)).to(sort_device)     # u64 order as i64 order
        if order is not None:
            k = k[order]
        _, idx = torch.sort(k, stable=True)
        order = idx if order is None else order[idx]
        del k, idx
    return order.cpu().numpy()


def _assert_sorted(words, what="rows out of canonical order"):
    """The gathered words are in lexicographic order: whatever sorted them, the order is checked here."""
    ok = words[-1][1:] >= words[-1][:-1]
    for w in reversed(words[:-1]):
        ok = (w[1:] > w[:-1]) | ((w[1:] == w[:-1]) & ok)
    assert ok.all(), what


def canonicalize(cols: dict, sort_device=None) -> dict:
    """``tad_oracle.canonicalize`` through the packed key words: result columns sorted by key columns, then flow_end."""
    words = _key_words(cols)
    order = _argsort_lex(words, sort_device)
    _assert_sorted(tuple(w[order] for w in words))
    return {k: np.asarray(v)[order] for k, v in cols.items()}


def reduce_max(values, starts):
    return np.maximum.reduceat(values, starts)


def reduce_sum(values, starts):
    """u64 sum of each duplicate run, wrapping mod 2^64 as ClickHouse's UInt64 sum (tad_oracle.py: run_job)."""
    return np.add.reduceat(values, starts)


# --------------------------------------------------------------------------------------------------------------------
# stages B and C
# --------------------------------------------------------------------------------------------------------------------
def _steps(sstart, slen):
    """(by_len, lens, base, counts): the series longest first, their lengths and first points; step i covers the
    series base[:counts[i]]."""
    by_len = np.argsort(-slen, kind="stable")
    lens = slen[by_len]
    counts = np.searchsorted(-lens, -np.arange(1, int(lens[0]) + 1), side="right")
    return by_len, lens, sstart[by_len], counts


def welford(x, lens, base, counts):
    """stddev_samp per series (longest first) by Spark's CentralMomentAgg: n += 1; d = x - avg; dn = d / n;
    avg += dn; m2 += d * (d - dn); sqrt(m2 / (n - 1)), NaN for one point."""
    avg = np.zeros(len(base))
    m2 = np.zeros(len(base))
    for i, c in enumerate(counts):
        d = x[base[:c] + i] - avg[:c]
        dn = d / float(i + 1)
        avg[:c] = avg[:c] + dn
        m2[:c] = m2[:c] + d * (d - dn)
    with np.errstate(invalid="ignore", divide="ignore"):
        sd = np.sqrt(m2 / (lens.astype(np.float64) - 1.0))
    sd[lens < 2] = np.nan
    return sd


def ewma(x, base, counts):
    """e_0 = 0; e_i = (1 - 0.5) e_{i-1} + 0.5 x_i, per point."""
    calc = np.empty(len(x))
    prev = np.zeros(len(base))
    for i, c in enumerate(counts):
        idx = base[:c] + i
        prev[:c] = 0.5 * prev[:c] + 0.5 * x[idx]
        calc[idx] = prev[:c]
    return calc


def ewma_flag(x, calc, sd_pt):
    """calculate_ewma_anomaly: strict ``|x - e| > stddev``; a NaN stddev (one point) flags nothing."""
    return np.abs(x - calc) > sd_pt


def brute_d2(xi, xj):
    """sklearn's brute-force squared distance, fl(fl(fl(xi xi) + fl(-2 fl(xi xj))) + fl(xj xj)), clipped at 0."""
    d = (xi * xi + (-2.0 * (xi * xj))) + xj * xj
    return np.where(d > 0.0, d, 0.0)


def _dbscan_small(x, sstart, slen, flag, chunk=1 << 16):
    """Series of at most 11 points: one padded 11 x 11 neighbourhood block each."""
    idx_s = np.flatnonzero(slen <= BRUTE_MAX_N)
    r2 = DBSCAN_EPS * DBSCAN_EPS
    k = np.arange(BRUTE_MAX_N)
    eye = np.eye(BRUTE_MAX_N, dtype=bool)
    for c0 in range(0, len(idx_s), chunk):
        s = idx_s[c0:c0 + chunk]
        valid = k[None, :] < slen[s][:, None]
        pos = np.where(valid, sstart[s][:, None] + k[None, :], 0)
        X = x[pos]
        with np.errstate(over="ignore", invalid="ignore"):
            nb = (brute_d2(X[:, :, None], X[:, None, :]) <= r2) | eye[None]
        nb &= valid[:, :, None] & valid[:, None, :]
        core = nb.sum(axis=2) >= DBSCAN_MIN_SAMPLES
        reach = (nb & core[:, None, :]).any(axis=2)
        flag[pos[valid]] = ~reach[valid]


def _dbscan_sweep(x, seg_start, seg_end, vorder, flag):
    """Series of 12 points and more, value-sorted: ``vorder`` lists their points series by series, each series in
    ascending value; ``seg_start`` / ``seg_end`` give every position of ``vorder`` its series' bounds in it."""
    v = x[vorder]
    n = len(v)
    pos = np.arange(n)
    eps = DBSCAN_EPS

    def within(off):
        """Position pos + off lies in the series and in the eps window of pos."""
        j = pos + off
        ok = (j >= seg_start) & (j < seg_end)
        jj = np.clip(j, 0, max(n - 1, 0))
        return ok & (np.abs(v - v[jj]) <= eps)

    left = [np.ones(n, bool)] + [within(-a) for a in range(1, DBSCAN_MIN_SAMPLES)]
    right = [np.ones(n, bool)] + [within(b) for b in range(1, DBSCAN_MIN_SAMPLES)]
    core = np.zeros(n, bool)
    for a in range(DBSCAN_MIN_SAMPLES):
        core |= left[a] & right[DBSCAN_MIN_SAMPLES - 1 - a]
    # nearest core at or before / at or after each position: by monotone rounding, if any core is in the window the
    # nearest one on that side is
    lc = np.maximum.accumulate(np.where(core, pos, -1)) if n else pos
    rc = np.minimum.accumulate(np.where(core, pos, n)[::-1])[::-1] if n else pos
    lok = lc >= seg_start
    rok = rc < seg_end
    reach = core.copy()
    reach |= lok & (np.abs(v - v[np.clip(lc, 0, max(n - 1, 0))]) <= eps)
    reach |= rok & (np.abs(v - v[np.clip(rc, 0, max(n - 1, 0))]) <= eps)
    flag[vorder] = ~reach


def dbscan_flags(values, x, sstart, slen, sort_device=None):
    flag = np.zeros(len(x), bool)
    _dbscan_small(x, sstart, slen, flag)
    big = slen > BRUTE_MAX_N
    if big.any():
        sid = np.repeat(np.arange(len(slen)), slen)
        pts = np.flatnonzero(big[sid])
        sub_sid = sid[pts]
        words = (sub_sid.astype(U64), values[pts])
        o = _argsort_lex(words, sort_device)
        _assert_sorted(tuple(w[o] for w in words), "points out of (series, value) order")
        vorder = pts[o]
        # series bounds within vorder: the big series, in series order, back to back
        bl = slen[big]
        bstart = np.cumsum(bl) - bl
        seg_start = np.repeat(bstart, bl)
        _dbscan_sweep(x, seg_start, seg_start + np.repeat(bl, bl), vorder, flag)
    return flag


# --------------------------------------------------------------------------------------------------------------------
# the job
# --------------------------------------------------------------------------------------------------------------------
def _columns(table, keep=None, names=_COLS):
    n = len(table["flow_end"])
    out = {}
    for c in names:
        a = table.get(c)
        a = np.zeros(n, dtype=_COLS[c]) if a is None else np.asarray(a, dtype=_COLS[c])
        out[c] = a if keep is None else a[keep]
    return out


def _empty():
    return {c: np.zeros(0, dtype=_out_dtype(c)) for c in OUT_COLUMNS}


def _run_piece(t, algo, reducer, emit_all, sort_device):
    n = len(t["flow_end"])
    if n == 0:
        return _empty(), 0, 0
    words = _key_words(t)
    order = _argsort_lex(words, sort_device)
    words = tuple(w[order] for w in words)
    _assert_sorted(words)
    w0, w1, w2 = words
    same_key = (w0[1:] == w0[:-1]) & (w1[1:] == w1[:-1]) & ((w2[1:] >> U64(32)) == (w2[:-1] >> U64(32)))
    same_point = same_key & (w2[1:] == w2[:-1])
    del w0, w1, words
    pstart = np.flatnonzero(np.concatenate(([True], ~same_point)))
    values = t["value"][order]
    values = (reduce_max if reducer == REDUCE_MAX else reduce_sum)(values, pstart)
    rows = order[pstart]                                   # one table row per point: its key columns and flow_end
    del order
    key_change = np.concatenate(([True], ~same_key))[pstart]
    del same_key, same_point
    sstart = np.flatnonzero(key_change)
    slen = np.diff(np.append(sstart, len(pstart)))
    x = values.astype(np.float64)                          # round to nearest even, as (double)u64

    by_len, lens, base, counts = _steps(sstart, slen)
    sd_sorted = welford(x, lens, base, counts)
    sd = np.empty(len(sstart))
    sd[by_len] = sd_sorted
    sd_pt = np.repeat(sd, slen)
    if algo == ALGO_EWMA:
        calc = ewma(x, base, counts)
        flag = ewma_flag(x, calc, sd_pt)
    elif algo == ALGO_DBSCAN:
        calc = np.zeros(len(x))
        flag = dbscan_flags(values, x, sstart, slen, sort_device)
    else:
        raise ValueError("the columnar oracle computes EWMA and DBSCAN")
    sel = np.arange(len(x)) if emit_all else np.flatnonzero(flag)
    src = rows[sel]
    out = {c: t[c][src] for c in ("src_ip", "src_port", "dst_ip", "dst_port", "proto", "flow_start", "flow_end")}
    out.update(stddev=sd_pt[sel], algo_calc=calc[sel], throughput=x[sel], anomaly=flag[sel].astype(np.uint8))
    return {c: np.ascontiguousarray(out[c], dtype=_out_dtype(c)) for c in OUT_COLUMNS}, len(sstart), len(pstart)


def run_job(table: dict, algo: int = ALGO_EWMA, reducer: int = REDUCE_MAX, start_time: int = 0, end_time: int = 0,
            emit_all: bool = False, sort_device=None, max_chunk_rows: int | None = None, workers: int = 1):
    """(cols, n_series, n_points) as ``c_oracle.run_job`` returns them, the rows in ``tad_oracle.canonicalize`` order.
    ``table``: column name -> 1-D numpy array (absent key columns are 0).  ``workers``: pieces computed at once (numpy
    releases the GIL in its array operations)."""
    n = len(table["flow_end"])
    keep = None
    if start_time or end_time:
        keep = np.ones(n, bool)
        if start_time:
            keep &= _columns(table, names=("flow_start",))["flow_start"] >= np.uint32(start_time)
        if end_time:
            keep &= _columns(table, names=("flow_end",))["flow_end"] < np.uint32(end_time)
    if max_chunk_rows is None or n <= max_chunk_rows:
        return _run_piece(_columns(table, keep), algo, reducer, emit_all, sort_device)
    # pieces by source address: every series lies in one piece, and pieces in ascending address order concatenate to
    # the canonical order
    src = _columns(table, names=("src_ip",))["src_ip"]
    edges = np.unique(np.quantile(src[:: max(1, n // 1_000_000)], np.linspace(0, 1, -(-n // max_chunk_rows) + 1)[1:-1],
                                  method="higher").astype(np.uint32))
    bounds = list(zip([None] + list(edges), list(edges) + [None]))

    def piece(lo_hi):
        lo, hi = lo_hi
        m = np.ones(n, bool) if keep is None else keep.copy()
        if lo is not None:
            m &= src >= lo
        if hi is not None:
            m &= src < hi
        rows = np.flatnonzero(m)
        del m
        return _run_piece(_columns(table, rows), algo, reducer, emit_all, sort_device)

    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(max_workers=max(1, workers)) as pool:
        outs = list(pool.map(piece, bounds))
    return ({c: np.concatenate([o[0][c] for o in outs]) for c in OUT_COLUMNS}, sum(o[1] for o in outs),
            sum(o[2] for o in outs))
