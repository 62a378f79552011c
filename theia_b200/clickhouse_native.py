"""ClickHouse ``Native`` format reader / writer for the columns the TAD job touches.

Replaces the JDBC transport of the reference job: ``spark.read.jdbc`` of the stage-A query
(anomaly_detection.py:655-662) and ``df.write.jdbc`` into ``tadetector`` (:713-726).  The shim issues the
same query with ``FORMAT Native`` (HTTP interface or clickhouse-go column blocks, go.mod:7) and feeds the byte
stream to :func:`read_native`; results go back as one ``INSERT INTO tadetector FORMAT Native`` body built by
:func:`write_native`.

Format (ClickHouse docs, "Native": *data is written and read by blocks in binary format; for each block the
number of columns, the number of rows, column names and types, and parts of columns in this block are recorded
one after another*), as restated here:

    block   := VarUInt n_columns, VarUInt n_rows, column * n_columns
    column  := String name, String type, data[n_rows]
    String  := VarUInt length, bytes
    data    := little-endian fixed-width values (UInt*/Int*/Float*, Date = UInt16, DateTime = UInt32,
               DateTime64 = Int64, IPv4 = UInt32), or n_rows Strings, or FixedString(N) = N bytes each,
               or Nullable(T) = n_rows null-flag bytes followed by T data

PARITY: unpinned -- there is no ClickHouse server or client in this image to produce golden bytes; the types are
the ones of ``flows`` / ``tadetector`` (create_table.sh:31-85, 363-384), none of which uses LowCardinality, arrays
or other composite serialisations (those raise ``NotImplementedError``).  tests/test_clickhouse_native.py pins
the byte layout with hand-assembled blocks.

Fixed-width columns are zero-copy ``numpy.frombuffer`` views; String columns are indexed by the library
(``tad_ch_string_index``), IPv4 text becomes the u32 key column there as well (``tad_ch_parse_ipv4``).
"""
from __future__ import annotations

import ctypes as C
import re

import numpy as np

from . import _lib

_FIXED = {
    "UInt8": "<u1", "UInt16": "<u2", "UInt32": "<u4", "UInt64": "<u8",
    "Int8": "<i1", "Int16": "<i2", "Int32": "<i4", "Int64": "<i8",
    "Float32": "<f4", "Float64": "<f8", "Date": "<u2", "DateTime": "<u4", "IPv4": "<u4", "Bool": "<u1",
}


class StringColumn:
    """A String column kept as (buffer, offsets, lengths): rows are decoded only when asked for."""

    def __init__(self, buf, offsets: np.ndarray, lengths: np.ndarray, start: int = 0, end: int | None = None):
        self.buf, self.offsets, self.lengths = buf, offsets, lengths
        self.start, self.end = start, end       # the column's byte span in ``buf`` (as read from a block)

    def __len__(self):
        return len(self.offsets)

    def __getitem__(self, i) -> str:
        o = int(self.offsets[i])
        return bytes(self.buf[o:o + int(self.lengths[i])]).decode("utf-8", "replace")

    def to_list(self) -> list:
        return [self[i] for i in range(len(self))]

    def to_numpy(self) -> np.ndarray:
        return np.asarray(self.to_list(), dtype=object)

    def ipv4(self):
        """(u32 values, is_ipv4 mask): dotted quads parsed by the library, everything else flagged for the dictionary."""
        n = len(self)
        out, ok = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint8)
        if n:
            base = np.frombuffer(self.buf, dtype=np.uint8)
            rc = _lib.load().tad_ch_parse_ipv4(base.ctypes.data, self.offsets.ctypes.data, self.lengths.ctypes.data, n,
                                              out.ctypes.data, ok.ctypes.data)
            if rc != 0:
                raise ValueError("tad_ch_parse_ipv4 failed (%d)" % rc)
        return out, ok.astype(bool)

    def text(self):
        """(column bytes, marks): the column exactly as it sits in its Native block, and the byte offset of rows 0, 32,
        64, ... in it -- a text key slot of ``StreamJob.push`` (tad_stream_push_text).  Both come from the index the
        reader already built."""
        end = self.end if self.end is not None else (int(self.offsets[-1]) + int(self.lengths[-1]) if len(self) else self.start)
        data = np.frombuffer(self.buf, dtype=np.uint8)[self.start:end]
        lens = self.lengths[::32].astype(np.uint64)
        vlen = np.ones(len(lens), dtype=np.uint64)
        for bits in (7, 14, 21, 28):
            vlen += lens >= np.uint64(1 << bits)
        return data, self.offsets[::32] - vlen - np.uint64(self.start)

    def codes(self):
        """(ids, names): dense dictionary ids in order of first appearance -- the shim's per-job string dictionary
        (hashing and comparison run in the library; only the distinct names become Python strings)."""
        n = len(self)
        ids, first = np.zeros(n, dtype=np.uint32), np.zeros(max(n, 1), dtype=np.uint64)
        nu = C.c_uint32(0)
        if n:
            base = np.frombuffer(self.buf, dtype=np.uint8)
            rc = _lib.load().tad_ch_dictionary(base.ctypes.data, self.offsets.ctypes.data, self.lengths.ctypes.data, n,
                                               ids.ctypes.data, first.ctypes.data, C.byref(nu))
            if rc != 0:
                raise ValueError("tad_ch_dictionary failed (%d)" % rc)
        return ids, [self[int(r)] for r in first[:nu.value]]


def _varuint(buf, p: int):
    n, shift = 0, 0
    while True:
        if p >= len(buf):
            raise ValueError("truncated Native block (VarUInt)")
        b = buf[p]
        p += 1
        n |= (b & 0x7F) << shift
        if not b & 0x80:
            return n, p
        shift += 7
        if shift > 63:
            raise ValueError("VarUInt longer than 64 bits")


def _string(buf, p: int):
    n, p = _varuint(buf, p)
    if p + n > len(buf):
        raise ValueError("truncated Native block (String)")
    return bytes(buf[p:p + n]).decode("utf-8"), p + n


def _read_data(buf, p: int, typ: str, rows: int):
    m = re.fullmatch(r"Nullable\((.*)\)", typ)
    if m:
        nulls = np.frombuffer(buf, dtype=np.uint8, count=rows, offset=p).astype(bool)
        vals, p = _read_data(buf, p + rows, m.group(1), rows)
        return (vals, nulls), p
    base = re.sub(r"\(.*\)$", "", typ)
    if base == "DateTime64":
        base_dt = "<i8"
    else:
        base_dt = _FIXED.get(base)
    if base_dt is not None and (base == typ or base in ("DateTime", "DateTime64")):
        dt = np.dtype(base_dt)
        if p + rows * dt.itemsize > len(buf):
            raise ValueError("truncated Native block (%s x %d)" % (typ, rows))
        return np.frombuffer(buf, dtype=dt, count=rows, offset=p), p + rows * dt.itemsize
    if typ == "String":
        offsets, lengths = np.zeros(rows, dtype=np.uint64), np.zeros(rows, dtype=np.uint32)
        used = C.c_size_t(0)
        view = np.frombuffer(buf, dtype=np.uint8)
        rc = _lib.load().tad_ch_string_index(view.ctypes.data + p, len(buf) - p, rows, offsets.ctypes.data, lengths.ctypes.data,
                                            C.byref(used))
        if rc != 0:
            raise ValueError("truncated or malformed String column")
        return StringColumn(buf, offsets + np.uint64(p), lengths, p, p + used.value), p + used.value
    m = re.fullmatch(r"FixedString\((\d+)\)", typ)
    if m:
        w = int(m.group(1))
        if p + rows * w > len(buf):
            raise ValueError("truncated Native block (%s)" % typ)
        return np.frombuffer(buf, dtype="S%d" % w, count=rows, offset=p), p + rows * w
    raise NotImplementedError("Native type %r is not used by flows / tadetector and is not decoded" % typ)


def read_blocks(data):
    """Yield one ``{name: column}`` dict (plus ``{name: type}``) per block of a Native byte stream."""
    buf = memoryview(data).cast("B") if not isinstance(data, memoryview) else data.cast("B")
    p = 0
    while p < len(buf):
        ncols, p = _varuint(buf, p)
        rows, p = _varuint(buf, p)
        if ncols > len(buf) - p or (ncols and rows > len(buf) - p):      # every column / value takes at least one byte
            raise ValueError("Native block header claims %d columns x %d rows in %d bytes" % (ncols, rows, len(buf) - p))
        cols, types = {}, {}
        for _ in range(ncols):
            name, p = _string(buf, p)
            typ, p = _string(buf, p)
            cols[name], p = _read_data(buf, p, typ, rows)
            types[name] = typ
        yield cols, types, rows


def _read_one_block(buf, p: int):
    """One block starting at ``p``: (cols, types, rows, next_p).  Raises ValueError when the buffer ends early."""
    ncols, p = _varuint(buf, p)
    rows, p = _varuint(buf, p)
    if ncols > len(buf) - p or (ncols and rows > len(buf) - p):
        raise ValueError("truncated Native block (header claims %d columns x %d rows in %d bytes)" % (ncols, rows, len(buf) - p))
    cols, types = {}, {}
    for _ in range(ncols):
        name, p = _string(buf, p)
        typ, p = _string(buf, p)
        cols[name], p = _read_data(buf, p, typ, rows)
        types[name] = typ
    return cols, types, rows, p


def read_blocks_stream(chunks):
    """Like :func:`read_blocks`, for a Native stream that arrives in pieces (an iterable of bytes objects, e.g. an HTTP body read
    4 MB at a time): a block is decoded as soon as its last byte is there, and the bytes of finished blocks are dropped, so the
    peak memory is one block plus one piece instead of the whole response.  The yielded columns own their data (copies; String
    columns keep a private copy of their block)."""
    pending = bytearray()
    it = iter(chunks)
    eof = False
    while True:
        if pending:
            try:
                snap = bytes(pending)                      # a stable buffer for the zero-copy views of this attempt
                cols, types, rows, used = _read_one_block(memoryview(snap), 0)
            except ValueError:
                if eof:
                    raise
            else:
                del pending[:used]
                yield {k: (v if isinstance(v, (StringColumn, tuple)) else np.array(v)) for k, v in cols.items()}, types, rows
                continue
        if eof:
            return
        try:
            piece = next(it)
        except StopIteration:
            eof = True
            if not pending:
                return
            continue
        pending += piece


def read_native(data) -> dict:
    """All blocks of a Native stream concatenated: ``{column: numpy array}`` (String columns as object arrays --
    use :func:`read_blocks` to keep them as :class:`StringColumn` and avoid materialising Python strings)."""
    parts, order = {}, []
    for cols, _types, _rows in read_blocks(data):
        for k, v in cols.items():
            if k not in parts:
                parts[k] = []
                order.append(k)
            if isinstance(v, tuple):                       # Nullable: masked values -> None
                vals, nulls = v
                vals = vals.to_numpy() if isinstance(vals, StringColumn) else np.asarray(vals).astype(object)
                vals[nulls] = None
                v = vals
            elif isinstance(v, StringColumn):
                v = v.to_numpy()
            parts[k].append(np.asarray(v))
    return {k: (np.concatenate(parts[k]) if len(parts[k]) > 1 else parts[k][0]) for k in order}


def flows_from_native(data) -> dict:
    """Native stream of the stage-A select -> the ``flows`` dict :func:`theia_b200.anomaly_detection.anomaly_detection`
    takes.  sourceIP / destinationIP become u32 where every value is a dotted quad (the common case: the engine's key
    columns are filled without creating a Python string per row); otherwise they stay strings for the dictionary.
    ``data``: the whole stream as bytes, or an iterable of pieces (decoded block by block as they arrive)."""
    parts, order = {}, []
    blocks = read_blocks(data) if isinstance(data, (bytes, bytearray, memoryview)) else read_blocks_stream(data)
    for cols, _types, _rows in blocks:
        for k, v in cols.items():
            if isinstance(v, StringColumn):
                if k in ("sourceIP", "destinationIP"):
                    ip, ok = v.ipv4()
                    v = ip if ok.all() else v.to_numpy()
                else:
                    v = v.to_numpy()
            elif isinstance(v, tuple):
                raise NotImplementedError("Nullable columns are not part of the flows schema")
            if k not in parts:
                parts[k] = []
                order.append(k)
            parts[k].append(np.asarray(v))
    out = {}
    for k in order:
        kinds = {a.dtype.kind for a in parts[k]}
        if k in ("sourceIP", "destinationIP") and len(kinds) > 1:          # mixed blocks: fall back to text
            from .anomaly_detection import u32_to_ip
            parts[k] = [a if a.dtype.kind == "O" else np.asarray([u32_to_ip(int(x)) for x in a], dtype=object) for a in parts[k]]
        out[k] = np.concatenate(parts[k]) if len(parts[k]) > 1 else parts[k][0]
    return out


# ---- writer -------------------------------------------------------------------------------------------------
def _enc_varuint(n: int) -> bytes:
    out = bytearray()
    while True:
        b = n & 0x7F
        n >>= 7
        if n:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _enc_string(s) -> bytes:
    b = s if isinstance(s, (bytes, bytearray)) else str(s).encode("utf-8")
    return _enc_varuint(len(b)) + bytes(b)


def write_native(columns) -> bytes:
    """One Native block from ``[(name, type, values), ...]``.  ``values`` of a String column may be a sequence of
    str / bytes, or a ``numpy.uint32`` array of IPv4 addresses (formatted as dotted quads by the library)."""
    columns = list(columns)
    rows = len(columns[0][2]) if columns else 0
    out = [_enc_varuint(len(columns)), _enc_varuint(rows)]
    for name, typ, vals in columns:
        if len(vals) != rows:
            raise ValueError("column %s has %d rows, expected %d" % (name, len(vals), rows))
        out.append(_enc_string(name))
        out.append(_enc_string(typ))
        base = re.sub(r"\(.*\)$", "", typ)
        if typ == "String":
            a = np.asarray(vals)
            if a.dtype.kind == "u" and a.dtype.itemsize == 4:
                ips = np.ascontiguousarray(a, dtype=np.uint32)
                buf = np.empty(16 * rows + 16, dtype=np.uint8)
                used = C.c_size_t(0)
                rc = _lib.load().tad_ch_format_ipv4(ips.ctypes.data, rows, buf.ctypes.data, buf.size, C.byref(used))
                if rc != 0:
                    raise ValueError("tad_ch_format_ipv4 failed (%d)" % rc)
                out.append(buf[:used.value].tobytes())
            else:
                out.append(b"".join(_enc_string(v) for v in vals))
        elif base in _FIXED and (base == typ or base == "DateTime"):
            out.append(np.ascontiguousarray(np.asarray(vals), dtype=_FIXED[base]).tobytes())
        else:
            raise NotImplementedError("Native type %r is not written" % typ)
    return b"".join(out)


TADETECTOR_SCHEMA = (              # create_table.sh:363-384, column order of the table
    ("sourceIP", "String"), ("sourceTransportPort", "UInt16"), ("destinationIP", "String"),
    ("destinationTransportPort", "UInt16"), ("protocolIdentifier", "UInt16"), ("flowStartSeconds", "DateTime"),
    ("podNamespace", "String"), ("podLabels", "String"), ("podName", "String"), ("destinationServicePortName", "String"),
    ("direction", "String"), ("flowEndSeconds", "DateTime"), ("throughputStandardDeviation", "Float64"),
    ("aggType", "String"), ("algoType", "String"), ("algoCalc", "Float64"), ("throughput", "Float64"),
    ("anomaly", "String"), ("id", "String"),
)


def tadetector_block(rows: list) -> bytes:
    """Result rows (the dicts :func:`theia_b200.anomaly_detection.anomaly_detection` returns) -> the body of
    ``INSERT INTO tadetector FORMAT Native``; columns a row does not carry take the table defaults ('' / 0), as
    the reference's partial-column JDBC append does (anomaly_detection.py:713-726)."""
    cols = []
    for name, typ in TADETECTOR_SCHEMA:
        if typ == "String":
            vals = [str(r.get(name, "")) for r in rows]
        elif typ == "Float64":
            vals = np.asarray([float("nan") if r.get(name) is None else float(r.get(name, 0.0)) for r in rows], dtype=np.float64)
            if name == "throughputStandardDeviation":
                vals = _null_to_default(vals)
        else:
            vals = np.asarray([_as_int(r.get(name, 0)) for r in rows], dtype=_FIXED[typ])
        cols.append((name, typ, vals))
    return write_native(cols)


def _null_to_default(stddev) -> np.ndarray:
    """stddev_samp of a single point is SQL NULL (NaN in the engine's result).  The reference's JDBC append writes NULL
    into the non-nullable Float64 column throughputStandardDeviation (create_table.sh:363-384), where it becomes the
    column default 0 -- so that is what goes into the block, not NaN."""
    a = np.asarray(stddev, dtype=np.float64)
    return np.where(np.isfinite(a), a, 0.0)


def _as_int(v) -> int:
    if hasattr(v, "timestamp"):
        return int(v.timestamp())
    if isinstance(v, str):                                   # the sentinel row's flowStartSeconds = now() as text (:397)
        from datetime import datetime
        return int(datetime.strptime(v, "%Y-%m-%d %H:%M:%S").timestamp())
    return int(v)


def _string_column_bytes(values=None, const=None, rows=0, ids=None, names=None) -> bytes:
    """Data bytes of a String column without a Python object per row: a constant repeated, or dictionary ids mapped to
    their pre-encoded names."""
    if const is not None:
        return _enc_string(const) * rows
    enc = np.empty(len(names), dtype=object)
    for i, nm in enumerate(names):
        enc[i] = _enc_string(nm)
    return b"".join(enc[np.asarray(ids, dtype=np.int64)].tolist())


class Names:
    """A dictionary as one byte array and offsets (``StreamJob.names``): the name of id k is data[offsets[k]:offsets[k+1]]."""

    def __init__(self, data, offsets):
        self.data = np.ascontiguousarray(data, dtype=np.uint8)
        self.offsets = np.ascontiguousarray(offsets, dtype=np.uint64)


def format_names(names: Names, ids) -> bytes:
    """String column bytes of ``names`` at ``ids`` (tad_ch_format_names): no Python object per name or row."""
    ids = np.ascontiguousarray(ids, dtype=np.uint32)
    count = len(names.offsets) - 1
    # capacity only: an id past the dictionary is rejected by the library call
    lens = np.diff(names.offsets)[np.minimum(ids, count - 1)] if len(ids) and count > 0 else np.zeros(1, dtype=np.uint64)
    cap = int(lens.sum()) + 10 * len(ids) + 1
    out = np.empty(cap, dtype=np.uint8)
    used = C.c_size_t(0)
    data = names.data if len(names.data) else np.zeros(1, dtype=np.uint8)
    rc = _lib.load().tad_ch_format_names(data.ctypes.data, names.offsets.ctypes.data, count, ids.ctypes.data, len(ids),
                                         out.ctypes.data, cap, C.byref(used))
    if rc != 0:
        raise ValueError("tad_ch_format_names failed (%d): an id past the dictionary" % rc)
    return out[:used.value].tobytes()


def tadetector_block_from_result(got: dict, plan, dicts: dict, algo_type: str, tad_id: str) -> bytes:
    """The same INSERT body as ``tadetector_block(_result_rows(...))`` (theia_b200/anomaly_detection.py), built column-wise
    from the engine's result arrays: no per-row dicts, so a job with millions of anomalous points stays array-speed.  The
    caller handles the empty result (sentinel row) through the row-wise path."""
    from .anomaly_detection import remove_meaningless_labels
    n = len(got["flow_end"])
    agg_type = plan.agg_flow if plan.agg_flow else "None"
    cols = {name: None for name, _ in TADETECTOR_SCHEMA}

    def ip_col(slot):
        d = dicts[slot]
        if isinstance(d, Names):                                # a device dictionary (text key slot)
            return ("names", got[slot], d)
        if d.names:                                             # the column went through the dictionary (non-IPv4 text)
            return ("ids", np.asarray(got[slot]), list(d.names))
        return ("ipv4", np.ascontiguousarray(got[slot], dtype=np.uint32), None)

    def name_col(slot):
        d = dicts[slot]
        if isinstance(d, Names):
            return ("names", got[slot], d)
        return ("ids", np.asarray(got[slot]), list(d.names))

    def labels_col(slot):
        d, ids = dicts[slot], np.asarray(got[slot])
        if isinstance(d, Names):                # cleaned once per distinct name the result uses
            used, inv = np.unique(ids, return_inverse=True)
            names = [remove_meaningless_labels(bytes(d.data[int(d.offsets[k]):int(d.offsets[k + 1])]).decode())
                     for k in used]
            return ("ids", inv.reshape(-1), names)
        return ("ids", ids, [remove_meaningless_labels(x) for x in d.names])

    if plan.agg_flow == "pod":
        cols["podNamespace"] = name_col("src_ip")
        if plan.branches[0].group[1] == "podLabels":
            cols["podLabels"] = labels_col("dst_ip")
        else:
            cols["podName"] = name_col("dst_ip")
        cols["direction"] = ("ids", (np.asarray(got["proto"]) != 0).astype(np.int64), ["inbound", "outbound"])
    elif plan.agg_flow == "external":
        cols["destinationIP"] = ip_col("dst_ip")
    elif plan.agg_flow == "svc":
        cols["destinationServicePortName"] = name_col("src_ip")
    else:
        cols["sourceIP"], cols["destinationIP"] = ip_col("src_ip"), ip_col("dst_ip")
        cols["sourceTransportPort"] = ("num", got["src_port"], None)
        cols["destinationTransportPort"] = ("num", got["dst_port"], None)
        cols["protocolIdentifier"] = ("num", got["proto"], None)
        cols["flowStartSeconds"] = ("num", got["flow_start"], None)
    cols["flowEndSeconds"] = ("num", got["flow_end"], None)
    cols["throughputStandardDeviation"] = ("num", _null_to_default(got["stddev"]), None)
    cols["algoCalc"] = ("num", got["algo_calc"], None)
    cols["throughput"] = ("num", got["throughput"], None)
    for name, v in (("aggType", agg_type), ("algoType", algo_type), ("anomaly", "true"), ("id", tad_id)):
        cols[name] = ("const", v, None)

    out = [_enc_varuint(len(TADETECTOR_SCHEMA)), _enc_varuint(n)]
    for name, typ in TADETECTOR_SCHEMA:
        out.append(_enc_string(name))
        out.append(_enc_string(typ))
        spec = cols[name]
        if typ == "String":
            if spec is None:
                out.append(b"\x00" * n)                          # '' : the table default
            elif spec[0] == "const":
                out.append(_string_column_bytes(const=spec[1], rows=n))
            elif spec[0] == "names":
                out.append(format_names(spec[2], spec[1]))
            elif spec[0] == "ipv4":
                buf = np.empty(16 * n + 16, dtype=np.uint8)
                used = C.c_size_t(0)
                if _lib.load().tad_ch_format_ipv4(spec[1].ctypes.data, n, buf.ctypes.data, buf.size, C.byref(used)) != 0:
                    raise ValueError("tad_ch_format_ipv4 failed")
                out.append(buf[:used.value].tobytes())
            else:
                out.append(_string_column_bytes(ids=spec[1], names=spec[2]))
        else:
            vals = np.zeros(n) if spec is None else np.asarray(spec[1])
            out.append(np.ascontiguousarray(vals, dtype=_FIXED[re.sub(r"\(.*\)$", "", typ)]).tobytes())
    return b"".join(out)

