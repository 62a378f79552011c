"""Host-side mirror of the reference job's interface (plugins/anomaly-detection/anomaly_detection.py),
on top of the C ABI.  What the Go shim of INTEGRATION.md does, written in the language the reference job
is written in, so the parity tests read like the reference's own tests.

reference                               here
--------------------------------------  ------------------------------------------------------------
generate_tad_sql_query (:507-614)       plan_query() -> QueryPlan: WHERE predicate, key columns, reducer;
                                        QueryPlan.to_sql() renders the reference's SQL text (pinned to
                                        the reference's 12 SQL test cases) for ClickHouse push-down
anomaly_detection (:647-710)            anomaly_detection(): plan -> host string predicates + dictionary
                                        encoding -> tad_submit / tad_wait / tad_result -> tadetector rows
filter_df_with_true_anomalies (:352-421) _result_rows(): per-aggregation column sets + the sentinel row
remove_meaningless_labels (:631-644)    remove_meaningless_labels()
main()/getopt (:729-900)                main() / parse_args(): same long options (and the controller's spelling
                                        --ns-ignore-list, which the reference's getopt rejects), same
                                        CH_USERNAME / CH_PASSWORD, same tables; ClickHouse is reached over the
                                        HTTP port of --db_jdbc_url with FORMAT Native (ClickHouseHTTP)
write_anomaly_detection_result (:713-726) clickhouse_native.tadetector_block() -> INSERT ... FORMAT Native

Flow tables are dicts of numpy arrays named like the ClickHouse ``flows`` columns
(build/charts/theia/provisioning/datasources/create_table.sh:31-85); IPs may be dotted strings or u32.
All numeric work happens on the GPU; strings never leave the host (they become dictionary ids).
"""
from __future__ import annotations

import calendar
import getopt
import json
import logging
import os
import re
import sys
import time
import uuid
from dataclasses import dataclass, field
from datetime import datetime

import numpy as np

from . import _lib as L

TABLE_NAME = "default.flows"
RESULT_TABLE_NAME = "default.tadetector"                                               # anomaly_detection.py:732
DEFAULT_JDBC_URL = "jdbc:clickhouse://clickhouse-clickhouse.flow-visibility.svc:8123"   # anomaly_detection.py:730-731
MEANINGLESS_LABELS = ("pod-template-hash", "controller-revision-hash", "pod-template-generation")
VALID_ALGOS = ("EWMA", "ARIMA", "DBSCAN")
KEY_SLOTS = ("src_ip", "src_port", "dst_ip", "dst_port", "proto", "flow_start")

# per-connection query (anomaly_detection.py:52-61, 109-116)
_CONN_SELECT = ["sourceIP", "sourceTransportPort", "destinationIP", "destinationTransportPort", "protocolIdentifier",
                "flowStartSeconds", "flowEndSeconds", "max(throughput)"]
_CONN_GROUP = ["sourceIP", "sourceTransportPort", "destinationIP", "destinationTransportPort", "protocolIdentifier",
               "flowStartSeconds"]


def remove_meaningless_labels(pod_labels: str) -> str:
    """anomaly_detection.py:631-644."""
    try:
        d = json.loads(pod_labels)
    except Exception:
        return ""
    return json.dumps({k: v for k, v in d.items() if k not in MEANINGLESS_LABELS}, sort_keys=True)


def _sql_list(names):
    return ", ".join("'{}'".format(x) for x in names)


@dataclass
class Branch:
    """One SELECT of the (possibly UNION ALL) stage-A query."""
    select: list
    where: list                      # SQL condition strings, joined by the caller
    group: list
    key: dict = field(default_factory=dict)      # key slot -> flows column (or ('const', code))
    direction: str = ""


@dataclass
class QueryPlan:
    agg_flow: str
    branches: list
    reducer: int
    ns_ignore: list
    start_time: str
    end_time: str
    pod_sql_extension: str = ""

    def to_sql(self) -> str:
        """The text generate_tad_sql_query returns (anomaly_detection.py:507-614)."""
        if self.agg_flow == "pod":
            parts = []
            for b in self.branches:
                parts.append("(SELECT {} FROM {} WHERE {} {} GROUP BY {}) ".format(
                    ", ".join(b.select), TABLE_NAME, b.where[0], self.pod_sql_extension, ", ".join(b.group)))
            return "SELECT * FROM " + "UNION ALL ".join(parts)
        b = self.branches[0]
        sql = "SELECT {} FROM {} ".format(", ".join(b.select), TABLE_NAME)
        if b.where:
            sql += "WHERE " + " AND ".join(b.where) + " "
        return sql + "GROUP BY {} ".format(", ".join(b.group))


def plan_query(start_time="", end_time="", ns_ignore_list=(), agg_flow=None, pod_label=None, external_ip=None,
               svc_port_name=None, pod_name=None, pod_namespace=None) -> QueryPlan:
    """Same decisions as generate_tad_sql_query, as data instead of text."""
    ns_ignore_list = list(ns_ignore_list or [])
    if agg_flow == "pod":
        second = "podLabels"
        if pod_label:
            inbound = "ilike(destinationPodLabels, '%{}%') ".format(pod_label)
            outbound = "ilike(sourcePodLabels, '%{}%')".format(pod_label)
            if pod_namespace:
                inbound += " AND destinationPodNamespace = '{}'".format(pod_namespace)
                outbound += " AND sourcePodNamespace = '{}'".format(pod_namespace)
        elif pod_name:
            inbound = "destinationPodName = '{}'".format(pod_name)
            outbound = "sourcePodName = '{}'".format(pod_name)
            if pod_namespace:
                inbound += " AND destinationPodNamespace = '{}'".format(pod_namespace)
                outbound += " AND sourcePodNamespace = '{}'".format(pod_namespace)
            second = "podName"
        else:
            inbound = "destinationPodLabels <> '' "
            outbound = "sourcePodLabels <> ''"
        src_second = "PodLabels" if second == "podLabels" else "PodName"
        ext = ("AND sourcePodNamespace NOT IN ({0}) AND destinationPodNamespace NOT IN ({0})".format(
            _sql_list(ns_ignore_list)) if ns_ignore_list else "")
        group = ["podNamespace", second, "direction", "flowEndSeconds"]
        branches = [
            Branch(["destinationPodNamespace AS podNamespace", "destination%s AS %s" % (src_second, second),
                    "'inbound' AS direction", "flowEndSeconds", "sum(throughput)"], [inbound], group,
                   {"src_ip": "destinationPodNamespace", "dst_ip": "destination" + src_second, "proto": ("const", 0)},
                   "inbound"),
            Branch(["sourcePodNamespace AS podNamespace", "source%s AS %s" % (src_second, second),
                    "'outbound' AS direction", "flowEndSeconds", "sum(throughput)"], [outbound], group,
                   {"src_ip": "sourcePodNamespace", "dst_ip": "source" + src_second, "proto": ("const", 1)},
                   "outbound"),
        ]
        return QueryPlan("pod", branches, L.TAD_REDUCE_SUM, ns_ignore_list, "", "", ext)

    where = []
    if ns_ignore_list:
        where.append("sourcePodNamespace NOT IN ({0}) AND destinationPodNamespace NOT IN ({0})".format(
            _sql_list(ns_ignore_list)))
    if start_time:
        where.append("flowStartSeconds >= '{}'".format(start_time))
    if end_time:
        where.append("flowEndSeconds < '{}'".format(end_time))
    if agg_flow == "external":
        where.append("flowType = 3")
        if external_ip:
            where.append("destinationIP = '{}'".format(external_ip))
        b = Branch(["destinationIP", "flowType", "flowEndSeconds", "sum(throughput)"], where,
                   ["destinationIP", "flowType", "flowEndSeconds"], {"dst_ip": "destinationIP", "proto": "flowType"})
        return QueryPlan("external", [b], L.TAD_REDUCE_SUM, ns_ignore_list, start_time, end_time)
    if agg_flow == "svc":
        where.append("destinationServicePortName = '{}'".format(svc_port_name) if svc_port_name
                     else "destinationServicePortName <> ''")
        b = Branch(["destinationServicePortName", "flowEndSeconds", "sum(throughput)"], where,
                   ["destinationServicePortName", "flowEndSeconds"], {"src_ip": "destinationServicePortName"})
        return QueryPlan("svc", [b], L.TAD_REDUCE_SUM, ns_ignore_list, start_time, end_time)
    b = Branch(list(_CONN_SELECT), where, _CONN_GROUP + ["flowEndSeconds"],
               {"src_ip": "sourceIP", "src_port": "sourceTransportPort", "dst_ip": "destinationIP",
                "dst_port": "destinationTransportPort", "proto": "protocolIdentifier", "flow_start": "flowStartSeconds"})
    return QueryPlan(agg_flow or "", [b], L.TAD_REDUCE_MAX, ns_ignore_list, start_time, end_time)


# ------------------------------------------------------------------------------------------------
def _epoch(ts: str) -> int:
    """'YYYY-MM-DD hh:mm:ss' (UTC, anomaly_detection.py:754-762) -> epoch seconds; '' -> 0."""
    return calendar.timegm(datetime.strptime(ts, "%Y-%m-%d %H:%M:%S").timetuple()) if ts else 0


def ip_to_u32(col) -> np.ndarray:
    a = np.asarray(col)
    if a.dtype.kind in "iu":
        return a.astype(np.uint32)
    n = len(a)
    out, ok = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint8)
    if n == 0:
        return out
    try:
        b = np.ascontiguousarray(a.astype("S"))            # fixed-width ASCII cells; non-ASCII text cannot be an IPv4 address
    except UnicodeEncodeError:
        raise ValueError("not an IPv4 address column")
    w = b.dtype.itemsize
    offsets = np.arange(n, dtype=np.uint64) * np.uint64(w)
    lengths = np.char.str_len(b).astype(np.uint32)
    rc = L.load().tad_ch_parse_ipv4(b.ctypes.data, offsets.ctypes.data, lengths.ctypes.data, n, out.ctypes.data, ok.ctypes.data)
    if rc != 0 or not ok.all():
        bad = a[int(np.argmin(ok))] if rc == 0 else "?"
        raise ValueError("not an IPv4 address: %r" % (bad,))
    return out


def encode_ip_column(col, dictionary: "Dictionary") -> np.ndarray:
    """Key column for sourceIP / destinationIP.  IPv4 text becomes its u32 value; a column that holds anything else
    (IPv6, as dual-stack clusters export it) is dictionary-encoded as a whole, so ids and addresses never mix in one
    key column -- the reference groups by the text, and any injective encoding groups identically."""
    a = np.asarray(col)
    if a.dtype.kind in "iu":
        return a.astype(np.uint32)
    try:
        return ip_to_u32(a)
    except ValueError:
        return dictionary.encode(a)


def u32_to_ip(v: int) -> str:
    return "%d.%d.%d.%d" % ((v >> 24) & 255, (v >> 16) & 255, (v >> 8) & 255, v & 255)


class Dictionary:
    """string -> dense id (and back); what the shim keeps per job for non-numeric key columns."""

    def __init__(self):
        self.ids, self.names = {}, []

    def encode(self, col) -> np.ndarray:
        """ids in order of first appearance; hash-based (pandas.factorize) so a 1e8-row column costs seconds, not minutes:
        only the distinct values are touched by Python code."""
        a = np.asarray(col)
        if len(a) == 0:
            return np.zeros(0, dtype=np.uint32)
        try:
            import pandas as pd
            codes, uniques = pd.factorize(a.astype(object) if a.dtype.kind != "O" else a, sort=False, use_na_sentinel=False)
        except (ImportError, TypeError):                     # no pandas (or one without use_na_sentinel): same result, row by row
            seen, codes, uniques = {}, np.empty(len(a), dtype=np.int64), []
            for i, s in enumerate(a):
                j = seen.get(s)
                if j is None:
                    j = seen[s] = len(uniques)
                    uniques.append(s)
                codes[i] = j
        remap = np.empty(len(uniques), dtype=np.uint32)
        for k, u in enumerate(uniques):
            u = str(u)
            j = self.ids.get(u)
            if j is None:
                j = self.ids[u] = len(self.names)
                self.names.append(u)
            remap[k] = j
        return remap[codes]

    def encode_block(self, col: "BlockText", idx) -> np.ndarray:
        """ids of the rows ``idx`` of one block's String column.  Only the block's distinct names that those rows use are
        looked up (or added), so a name keeps its id across blocks and rounds and no Python string is made per row."""
        sel = col.ids[idx]
        used = np.zeros(len(col.names), dtype=bool)
        used[sel] = True
        remap = np.zeros(len(col.names), dtype=np.uint32)
        for k in np.flatnonzero(used):
            u = col.names[k]
            j = self.ids.get(u)
            if j is None:
                j = self.ids[u] = len(self.names)
                self.names.append(u)
            remap[k] = j
        return remap[sel]


class BlockText:
    """A String column of one Native block as the library's per-block dictionary (``StringColumn.codes()``): ``ids`` per
    row and the block's distinct ``names``.  Predicates and the job's Dictionary only ever look at the names."""

    def __init__(self, col):
        self.ids, names = col.codes()
        self.names = names

    def __len__(self):
        return len(self.ids)


def _text_test(col, test) -> np.ndarray:
    """``test`` (a vectorised predicate over a numpy str array) for every row of a text column: applied to the column
    itself, or for a BlockText to its distinct names and spread to the rows through the ids."""
    if isinstance(col, BlockText):
        return test(np.asarray(col.names, dtype=str))[col.ids]
    return test(np.asarray(col).astype(str))


def _host_mask(flows: dict, plan: QueryPlan, branch: Branch, pod_label, pod_name, pod_namespace, external_ip,
               svc_port_name) -> np.ndarray:
    """String predicates of the WHERE clause (time window and namespace ignore list run on the GPU)."""
    n = len(flows["flowEndSeconds"])
    m = np.ones(n, dtype=bool)
    if plan.agg_flow == "pod":
        side = "destination" if branch.direction == "inbound" else "source"
        if pod_label:
            m &= _text_test(flows[side + "PodLabels"],
                            lambda lab: np.char.find(np.char.lower(lab), pod_label.lower()) >= 0)   # ilike '%label%'
        elif pod_name:
            m &= _text_test(flows[side + "PodName"], lambda s: s == pod_name)
        else:
            m &= _text_test(flows[side + "PodLabels"], lambda s: s != "")
        if pod_namespace and (pod_label or pod_name):
            m &= _text_test(flows[side + "PodNamespace"], lambda s: s == pod_namespace)
    elif plan.agg_flow == "external":
        m &= np.asarray(flows["flowType"]) == 3
        if external_ip:
            dst = flows["destinationIP"]
            if not isinstance(dst, BlockText) and np.asarray(dst).dtype.kind in "iu":   # u32 key column (Native transport)
                try:
                    m &= np.asarray(dst) == ip_to_u32([external_ip])[0]
                except ValueError:
                    m &= False                                        # an IPv6 literal never equals an IPv4 column
            else:
                m &= _text_test(dst, lambda s: s == external_ip)      # destinationIP = '...' (:590-592)
    elif plan.agg_flow == "svc":
        m &= _text_test(flows["destinationServicePortName"], (lambda s: s == svc_port_name) if svc_port_name
                        else (lambda s: s != ""))
    if plan.start_time and "flow_start" not in branch.key and flows.get("flowStartSeconds") is not None:
        # external / svc: flowStartSeconds >= start is a WHERE condition (anomaly_detection.py:581-583) on a column
        # that is not part of the key, so it cannot ride the engine's key column: filter here.  A table that does
        # not carry the column came from raw_select_sql, whose WHERE clause already applied the same condition.
        m &= np.asarray(flows["flowStartSeconds"]).astype(np.int64) >= _epoch(plan.start_time)
    return m


def _dictionary_ids(col, idx, dictionary: Dictionary) -> np.ndarray:
    if isinstance(col, BlockText):
        return dictionary.encode_block(col, idx)
    return dictionary.encode(np.asarray(col)[idx])


def _branch_columns(flows: dict, plan: QueryPlan, br: Branch, masks: tuple, dicts: dict, ns_dict: Dictionary,
                    ipv4_as_u32: bool, text_slots=(), keep_all: bool = False) -> dict:
    """One branch's engine columns from a flows table or one block of it: the host predicates, then key slots,
    ``flow_end`` / ``value`` and, with an ignore list and ``ns_dict``, the namespace ids.  ``ipv4_as_u32``: an address column of IPv4 text
    becomes its u32 value (a whole table); otherwise text addresses go through the dictionary like every other String
    key, which keeps a name's id the same in every block of a stream.  ``text_slots``: key slots the engine encodes from
    the block's text itself (left None here).  ``keep_all``: every row, the host predicates left to the engine."""
    if keep_all:
        idx = np.arange(len(flows["flowEndSeconds"]))
    else:
        idx = np.flatnonzero(_host_mask(flows, plan, br, *masks))
    cols = {}
    for slot in KEY_SLOTS:
        src = br.key.get(slot)
        if src is None or slot in text_slots:
            cols[slot] = None
        elif isinstance(src, tuple):
            cols[slot] = np.full(len(idx), src[1], dtype=np.uint32)
        elif isinstance(flows[src], BlockText):
            cols[slot] = dicts[slot].encode_block(flows[src], idx)
        else:
            raw = np.asarray(flows[src])[idx]
            if src in ("sourceIP", "destinationIP") and ipv4_as_u32:
                cols[slot] = encode_ip_column(raw, dicts[slot])
            elif raw.dtype.kind in "iu":
                cols[slot] = raw
            else:
                cols[slot] = dicts[slot].encode(raw)
    cols["flow_end"] = np.asarray(flows["flowEndSeconds"])[idx]
    cols["value"] = np.asarray(flows["throughput"])[idx]
    if plan.ns_ignore and ns_dict is not None:
        cols["src_ns"] = _dictionary_ids(flows["sourcePodNamespace"], idx, ns_dict)
        cols["dst_ns"] = _dictionary_ids(flows["destinationPodNamespace"], idx, ns_dict)
    return cols


def anomaly_detection(engine, algo_type: str, flows: dict, start_time: str = "", end_time: str = "", tad_id: str = "",
                      ns_ignore_list=(), agg_flow=None, pod_label=None, external_ip=None, svc_port_name=None,
                      pod_name=None, pod_namespace=None, now=None, on_job=None):
    """anomaly_detection.py:647-710 + write_anomaly_detection_result (:713-726): returns the list of row dicts the
    reference appends to default.tadetector (one sentinel row when nothing is anomalous) and the job status."""
    got, st, plan, dicts = run_engine(engine, algo_type, flows, start_time, end_time, tad_id, ns_ignore_list, agg_flow, pod_label,
                                      external_ip, svc_port_name, pod_name, pod_namespace, on_job=on_job)
    return _result_rows(got, plan, dicts, algo_type, tad_id, pod_label, now), st


def run_engine(engine, algo_type: str, flows: dict, start_time: str = "", end_time: str = "", tad_id: str = "",
               ns_ignore_list=(), agg_flow=None, pod_label=None, external_ip=None, svc_port_name=None,
               pod_name=None, pod_namespace=None, on_job=None):
    """Everything of :func:`anomaly_detection` up to the engine's result arrays: (result SoA, status, plan, dictionaries).
    The job entry point builds its INSERT body from these column-wise instead of materialising a dict per row."""
    if algo_type not in VALID_ALGOS:
        raise ValueError("Algorithm should be in {}".format(" or ".join(VALID_ALGOS)))      # :811-818
    plan = plan_query(start_time, end_time, ns_ignore_list, agg_flow, pod_label, external_ip, svc_port_name, pod_name,
                      pod_namespace)
    dicts = {slot: Dictionary() for slot in KEY_SLOTS}
    ns_dict = Dictionary()
    masks = (pod_label, pod_name, pod_namespace, external_ip, svc_port_name)
    parts = [_branch_columns(flows, plan, br, masks, dicts, ns_dict, ipv4_as_u32=True) for br in plan.branches]
    table = {}
    for k in parts[0]:
        if any(p[k] is None for p in parts):
            table[k] = None
        else:
            table[k] = np.concatenate([np.asarray(p[k]) for p in parts])
    ignore_ids = [ns_dict.ids[n] for n in plan.ns_ignore if n in ns_dict.ids]
    # The engine applies ``flowStartSeconds >= start`` to its flow_start KEY column.  In the external / svc modes
    # flowStartSeconds is not a key (anomaly_detection.py:568-571), so the window's lower bound was applied above
    # (_host_mask, or already by the WHERE clause of the SELECT the job entry sends) and must not reach the GPU, whose
    # absent flow_start column reads as 0.
    start = _epoch(plan.start_time) if table.get("flow_start") is not None else 0
    kw = {} if on_job is None else {"on_job": on_job}      # progress hook of the controller (tad_poll while the job runs)
    got, st = engine.run(table, algo=algo_type, reducer=plan.reducer, start_time=start,
                         end_time=_epoch(plan.end_time), tad_id=tad_id, ns_ignore=ignore_ids, **kw)
    return got, st, plan, dicts


def _block_table(block: dict) -> dict:
    """A decoded Native block (``{column: numpy array or StringColumn}``) with every String column as a BlockText."""
    out = {}
    for k, v in block.items():
        if isinstance(v, tuple):
            raise NotImplementedError("Nullable columns are not part of the flows schema")
        out[k] = BlockText(v) if hasattr(v, "codes") else v
    return out


def run_engine_stream(engine, algo_type: str, blocks, start_time: str = "", end_time: str = "", tad_id: str = "",
                      ns_ignore_list=(), agg_flow=None, pod_label=None, external_ip=None, svc_port_name=None,
                      pod_name=None, pod_namespace=None, rows_hint: int = 0, on_job=None, device_text: bool = False,
                      device_ns: bool = False):
    """:func:`run_engine` over streamed input: ``blocks()`` yields one round of decoded Native blocks
    (``{column: numpy array or clickhouse_native.StringColumn}``, as ``read_blocks`` / ``read_blocks_stream`` yield them)
    and is called again for every round the engine asks for.  Each block's branches are pushed as they are built (two
    blocks per source block in ``pod`` mode); blocks are never concatenated, and only the engine's one block of
    look-ahead stays referenced.  String keys, text addresses included, go through the job's dictionaries, so a value has
    the same id in every block and round; the namespace dictionary starts with the ignore list, whose ids the job spec
    needs at submit.  ``rows_hint``: one round's rows (0 = unknown).  Returns (result SoA, status, plan, dictionaries).

    ``device_text``: in connection mode, the two address columns go to the engine as the block's String column bytes
    (``StringColumn.text()``, tad_stream_push_text) and are dictionary-encoded on the GPU; their dictionaries come back
    as ``clickhouse_native.Names`` (tad_job_names).  Connection mode is the one mode whose host mask keeps every row and
    reads no key text; with ``device_text=True`` the pod / svc / external modes keep their host encoding.
    ``device_text="all"``: those modes push their String keys as text too, every row of a block, and the engine
    evaluates their string predicates on the GPU (tad_submit_stream_filtered; :func:`_device_text_branches`).

    ``device_ns``: a job with an ignore list pushes the two namespace columns as text (``src_ns`` / ``dst_ns``,
    tad_stream_push_text_ns) and gives the list as names (tad_submit_stream_filtered_ns): the GPU tests every row's
    namespaces against it, and no namespace column is decoded or dictionary-encoded here.  That needs every row of a
    block pushed (connection mode, and the modes ``device_text="all"`` takes as text) and a list of names the GPU
    compares as the host path does (:func:`_ns_names_on_device`); otherwise the namespaces keep their host encoding."""
    from .clickhouse_native import Names
    if algo_type not in VALID_ALGOS:
        raise ValueError("Algorithm should be in {}".format(" or ".join(VALID_ALGOS)))
    plan = plan_query(start_time, end_time, ns_ignore_list, agg_flow, pod_label, external_ip, svc_port_name, pod_name,
                      pod_namespace)
    dicts = {slot: Dictionary() for slot in KEY_SLOTS}
    ignore = [str(x) for x in plan.ns_ignore]
    masks = (pod_label, pod_name, pod_namespace, external_ip, svc_port_name)
    # as in run_engine: the window's lower bound reaches the engine only through a flow_start key column
    start = _epoch(plan.start_time) if all("flow_start" in br.key for br in plan.branches) else 0
    branch_text, text_filter = [{} for _ in plan.branches], None
    head, rest = [], None
    if device_text == "all":
        # the first round's first block is read before the submit: whether the mode's keys can go as text depends on it
        rest = iter(blocks())
        head.append(next(rest, None))
        branch_text, text_filter = _device_text_branches(plan, head[0], *masks)
    elif device_text and not plan.agg_flow:
        branch_text = [{"src_ip": "sourceIP", "dst_ip": "destinationIP"}]
    # every row of a block is pushed in connection mode (its host mask keeps them all) and where the engine takes the
    # mode's predicates: only then can a block's namespace text stand for the rows pushed
    ns_text = bool(device_ns and ignore and (not plan.agg_flow or text_filter is not None) and _ns_names_on_device(ignore))
    ns_cols = {"src_ns": "sourcePodNamespace", "dst_ns": "destinationPodNamespace"} if ns_text else {}
    text_cols = {c for bt in branch_text for c in bt.values()} | set(ns_cols.values())
    if ns_text:
        ns_dict, ignore_ids, ns_kw = None, [], {"ns_ignore_names": [x.encode() for x in ignore]}
    else:
        # the namespace dictionary starts with the ignore list, whose ids the job spec needs at submit
        ns_dict, ns_kw = Dictionary(), {}
        ns_dict.encode(np.asarray(ignore, dtype=object))
        ignore_ids = sorted({ns_dict.ids[x] for x in ignore})

    def round0():
        while head:
            b = head.pop()
            if b is not None:
                yield b
        yield from (blocks() if rest is None else rest)

    # without namespace text, the namespace columns of an ignore list stay host-encoded, also where they are a text key
    host_cols = {"sourcePodNamespace", "destinationPodNamespace"} if plan.ns_ignore and not ns_text else set()
    pushed_text = False
    kw = {} if text_filter is None else {"text_filter": text_filter}
    job = engine.submit_stream(algo=algo_type, reducer=plan.reducer, start_time=start, end_time=_epoch(plan.end_time),
                               tad_id=tad_id, ns_ignore=ignore_ids, rows_hint=int(rows_hint), **kw, **ns_kw)
    if on_job is not None:
        on_job(job)
    try:
        rounds, again = 0, True
        while again:
            for block in (round0() if rounds == 0 else blocks()):
                raw = {c: block[c] for c in text_cols}
                flows = _block_table({k: v for k, v in block.items() if k not in text_cols or k in host_cols})
                del block
                for br, bt in zip(plan.branches, branch_text):
                    slots = {slot: raw[c] for slot, c in bt.items()}
                    cols = _branch_columns(flows, plan, br, masks, dicts, ns_dict, ipv4_as_u32=False, text_slots=slots,
                                           keep_all=text_filter is not None)
                    if len(cols["flow_end"]):
                        if slots or ns_cols:
                            job.push(cols, text={slot: raw[c].text() for slot, c in {**bt, **ns_cols}.items()})
                            pushed_text = pushed_text or bool(slots)
                        else:
                            job.push(cols)
                    del cols
                del flows
            again = job.end()
            rounds += 1
        st = job.wait()
        st["rounds"] = rounds
        got = job.result()
        if pushed_text:
            for slot in {s for bt in branch_text for s in bt}:
                dicts[slot] = Names(*job.names(slot))
    except BaseException:
        job.cancel()
        raise
    finally:
        if on_job is not None:
            on_job(None)
        job.release()
    return got, st, plan, dicts


def _ns_names_on_device(names) -> bool:
    """Whether the GPU's byte equality lists the same rows as the host path for these ignore-list names.  The host path
    compares the names with namespaces decoded as UTF-8 with errors replaced, so a name holding U+FFFD would also list
    the namespaces whose bytes are not UTF-8; a name that is not valid Unicode (a lone surrogate from the JSON list)
    has no bytes.  Both keep the host encoding; Kubernetes namespace names are ASCII."""
    for x in names:
        if "\ufffd" in x:
            return False
        try:
            x.encode("utf-8")
        except UnicodeEncodeError:
            return False
    return True


def _device_text_branches(plan: QueryPlan, first, pod_label, pod_name, pod_namespace, external_ip, svc_port_name):
    """``device_text="all"``: per branch the key slots the engine takes as text ({slot: flows column}) and the job's row
    predicates (engine.submit_stream's ``text_filter``; None in connection mode, which has none).  A mode whose
    conditions the engine cannot express keeps its host encoding (no text, no predicates): a non-ASCII ``--pod-label``
    (the GPU's ILIKE folds ASCII patterns only), or blocks that carry ``flowStartSeconds`` where it is not a key (its
    lower bound is a host predicate then; ``first`` is the job's first block, None for an empty round)."""
    host = [{} for _ in plan.branches], None
    if not plan.agg_flow:
        return [{"src_ip": "sourceIP", "dst_ip": "destinationIP"}], None
    if plan.start_time and first is not None and "flowStartSeconds" in first and \
            any("flow_start" not in br.key for br in plan.branches):
        return host
    if plan.agg_flow == "external":
        flt = {"proto_eq": 3}
        if external_ip:
            flt["dst_ip"] = ("eq", external_ip.encode())
        return [{"dst_ip": "destinationIP"}], flt
    if plan.agg_flow == "svc":
        return [{"src_ip": "destinationServicePortName"}], \
            {"src_ip": ("eq", svc_port_name.encode()) if svc_port_name else ("nonempty", b"")}
    if pod_label and not pod_label.isascii():
        return host
    if pod_label:
        flt = {"dst_ip": ("icontains", pod_label.encode())}
    elif pod_name:
        flt = {"dst_ip": ("eq", pod_name.encode())}
    else:
        flt = {"dst_ip": ("nonempty", b"")}
    if pod_namespace and (pod_label or pod_name):
        flt["src_ip"] = ("eq", pod_namespace.encode())
    return [{"src_ip": br.key["src_ip"], "dst_ip": br.key["dst_ip"]} for br in plan.branches], flt


def _ip_text(dictionary: "Dictionary", v: int) -> str:
    """Inverse of encode_ip_column: a column that went through the dictionary comes back through it."""
    return dictionary.names[v] if dictionary.names else u32_to_ip(v)


def _result_rows(got: dict, plan: QueryPlan, dicts: dict, algo_type: str, tad_id: str, pod_label, now=None) -> list:
    """filter_df_with_true_anomalies' projections (anomaly_detection.py:359-393), the string cast of ``anomaly``
    (:500-502), the ``id`` column (:503) and the sentinel row (:395-420)."""
    agg_type = plan.agg_flow if plan.agg_flow else "None"
    rows = []
    for i in range(len(got["flow_end"])):
        common = {"aggType": agg_type, "flowEndSeconds": int(got["flow_end"][i]),
                  "throughputStandardDeviation": float(got["stddev"][i]), "algoType": algo_type,
                  "algoCalc": float(got["algo_calc"][i]), "throughput": float(got["throughput"][i]),
                  "anomaly": "true", "id": tad_id}
        if plan.agg_flow == "pod":
            second = dicts["dst_ip"].names[int(got["dst_ip"][i])]
            row = {"podNamespace": dicts["src_ip"].names[int(got["src_ip"][i])],
                   "direction": "inbound" if int(got["proto"][i]) == 0 else "outbound"}
            if plan.branches[0].group[1] == "podLabels":
                row["podLabels"] = remove_meaningless_labels(second)          # :687-695
            else:
                row["podName"] = second
        elif plan.agg_flow == "external":
            row = {"destinationIP": _ip_text(dicts["dst_ip"], int(got["dst_ip"][i]))}
        elif plan.agg_flow == "svc":
            row = {"destinationServicePortName": dicts["src_ip"].names[int(got["src_ip"][i])]}
        else:
            row = {"sourceIP": _ip_text(dicts["src_ip"], int(got["src_ip"][i])), "sourceTransportPort": int(got["src_port"][i]),
                   "destinationIP": _ip_text(dicts["dst_ip"], int(got["dst_ip"][i])),
                   "destinationTransportPort": int(got["dst_port"][i]), "protocolIdentifier": int(got["proto"][i]),
                   "flowStartSeconds": int(got["flow_start"][i])}
        row.update(common)
        rows.append(row)
    if not rows:
        rows.append({
            "sourceIP": "None", "sourceTransportPort": 0, "destinationIP": "None", "destinationTransportPort": 0,
            "protocolIdentifier": 0,
            "flowStartSeconds": (now or datetime.now()).strftime("%Y-%m-%d %H:%M:%S"),
            "podNamespace": "None", "podLabels": "None", "podName": "None", "destinationServicePortName": "None",
            "direction": "None", "flowEndSeconds": 0, "throughputStandardDeviation": 0, "aggType": agg_type,
            "algoType": algo_type, "algoCalc": 0.0, "throughput": 0.0, "anomaly": "NO ANOMALY DETECTED", "id": tad_id})
    return rows


def parse_args(argv):
    """The job's command line (anomaly_detection.py:781-870).  Accepts the reference's long options AND the
    spelling the controller actually passes (--ns-ignore-list, controller.go:546), which the reference's
    getopt rejects with exit code 2 -- a reference bug this engine does not reproduce."""
    opts, _ = getopt.getopt(argv, "ht:d:s:e:i:n:f:l:x:p:N:P:", [
        "help", "algo=", "db_jdbc_url=", "start_time=", "end_time=", "id=", "ns_ignore_list=", "ns-ignore-list=",
        "agg-flow=", "pod-label=", "external-ip=", "svc-port-name=", "pod-name=", "pod-namespace="])
    out = {"algo": "", "db_jdbc_url": DEFAULT_JDBC_URL, "start_time": "", "end_time": "", "id": None, "ns_ignore_list": [], "agg_flow": "",
           "pod_label": "", "external_ip": "", "svc_port_name": "", "pod_name": "", "pod_namespace": ""}
    for opt, arg in opts:
        if opt in ("-a", "--algo"):
            if arg not in VALID_ALGOS:
                raise SystemExit(2)
            out["algo"] = arg
        elif opt in ("-s", "--start_time", "-e", "--end_time"):
            try:
                datetime.strptime(arg, "%Y-%m-%d %H:%M:%S")
            except ValueError:
                raise SystemExit(2)
            out["start_time" if opt in ("-s", "--start_time") else "end_time"] = arg
        elif opt in ("-n", "--ns_ignore_list", "--ns-ignore-list"):
            lst = json.loads(arg)
            if not isinstance(lst, list):
                raise SystemExit(2)
            out["ns_ignore_list"] = lst
        elif opt in ("-i", "--id"):
            out["id"] = arg
        elif opt in ("-d", "--db_jdbc_url"):
            out["db_jdbc_url"] = arg
        elif opt in ("-f", "--agg-flow"):
            out["agg_flow"] = arg
        elif opt in ("-l", "--pod-label"):
            out["pod_label"] = arg
        elif opt in ("-N", "--pod-name"):
            out["pod_name"] = arg
        elif opt in ("-P", "--pod-namespace"):
            out["pod_namespace"] = arg
        elif opt in ("-x", "--external-ip"):
            out["external_ip"] = arg
        elif opt in ("-p", "--svc-port-name"):
            out["svc_port_name"] = arg
    return out


def timed_job(engine, *args, **kw):
    """main()'s only timing hook: 'Anomaly Detection completed, id: {}, in {} seconds' (anomaly_detection.py:872-899)."""
    t0 = time.time()
    rows, st = anomaly_detection(engine, *args, **kw)
    return rows, st, time.time() - t0


# ------------------------------------------------------------------------------------------------
# the job's entry point: same argv, same environment, same tables as the reference's main()
# ------------------------------------------------------------------------------------------------
logger = logging.getLogger("anomaly_detection")


class ClickHouseError(RuntimeError):
    """A query ClickHouse rejected (exception code + the server's text)."""

    def __init__(self, code: int, text: str):
        super().__init__("ClickHouse exception %d: %s" % (code, text))
        self.code, self.text = code, text


def _is_ipv4_pushdown_failure(e: Exception) -> bool:
    """Only a failure of IPv4StringToNum itself (a non-IPv4 address in the table) justifies the second, text-mode scan;
    authentication, network and syntax errors must surface."""
    import urllib.error
    text = ""
    if isinstance(e, ClickHouseError):
        text = e.text
    elif isinstance(e, urllib.error.HTTPError):
        try:
            text = e.read(2000).decode(errors="replace")
        except Exception:
            text = str(e)
    else:
        text = str(e) if "DB::Exception" in str(e) else ""
    return any(k in text for k in ("IPv4StringToNum", "Invalid IPv4", "CANNOT_PARSE_IPV4", "Cannot parse IPv4", "Code: 441"))


class ClickHouseHTTP:
    """ClickHouse over its HTTP interface.  The reference hands its JDBC URL to the ClickHouse JDBC driver
    (anomaly_detection.py:655-662, 720-726), which talks to that very HTTP port (8123 in the default URL, :730-731);
    here the same host:port receives the query with ``FORMAT Native`` and the column blocks come back as bytes.
    Credentials: CH_USERNAME / CH_PASSWORD from the environment, as the reference reads them (:659-660)."""

    def __init__(self, jdbc_url: str = DEFAULT_JDBC_URL, user=None, password=None, timeout: float = 3600.0):
        rest = jdbc_url
        for prefix in ("jdbc:clickhouse://", "jdbc:ch://", "clickhouse://", "http://"):
            if rest.startswith(prefix):
                rest = rest[len(prefix):]
                break
        hostport, _, tail = rest.partition("/")
        self.base = "http://" + hostport + "/"
        self.database = tail.split("?")[0]
        self.user = os.getenv("CH_USERNAME") if user is None else user
        self.password = os.getenv("CH_PASSWORD") if password is None else password
        self.timeout = timeout

    def _post(self, query: str, body: bytes = b"") -> bytes:
        import urllib.parse
        import urllib.request
        # wait_end_of_query: ClickHouse buffers the response and reports a failure as a non-200 status instead of appending
        # an exception text to a 200 stream that would then be parsed as a column block
        params = {"query": query, "wait_end_of_query": "1"}
        if self.database:
            params["database"] = self.database
        req = urllib.request.Request(self.base + "?" + urllib.parse.urlencode(params), data=body, method="POST")
        if self.user:
            req.add_header("X-ClickHouse-User", self.user)
        if self.password:
            req.add_header("X-ClickHouse-Key", self.password)
        with urllib.request.urlopen(req, timeout=self.timeout) as resp:
            code = resp.headers.get("X-ClickHouse-Exception-Code")
            body = resp.read()
            if code not in (None, "", "0"):
                raise ClickHouseError(int(code), body[:500].decode(errors="replace"))
            return body

    def select_native(self, sql: str) -> bytes:
        return self._post(sql.rstrip() + " FORMAT Native")

    def select_native_stream(self, sql: str, piece: int = 4 << 20):
        """The same SELECT as a generator of byte pieces, decoded block by block by the caller while the rest is still on the
        wire.  No ``wait_end_of_query`` here (it would make the server buffer a multi-gigabyte result before the first byte):
        a failure before the first block shows in the status / exception header, one in mid-stream as ClickHouse's
        ``Code: N. DB::Exception: ...`` text at the end of the body, which is raised as :class:`ClickHouseError`."""
        import urllib.parse
        import urllib.request
        params = {"query": sql.rstrip() + " FORMAT Native"}
        if self.database:
            params["database"] = self.database
        req = urllib.request.Request(self.base + "?" + urllib.parse.urlencode(params), data=b"", method="POST")
        if self.user:
            req.add_header("X-ClickHouse-User", self.user)
        if self.password:
            req.add_header("X-ClickHouse-Key", self.password)
        with urllib.request.urlopen(req, timeout=self.timeout) as resp:
            code = resp.headers.get("X-ClickHouse-Exception-Code")
            if code not in (None, "", "0"):
                raise ClickHouseError(int(code), resp.read(2000).decode(errors="replace"))
            tail = b""
            while True:
                b = resp.read(piece)
                if not b:
                    break
                tail = (tail + b)[-600:]
                yield b
            i = tail.rfind(b"DB::Exception")
            if i >= 0:
                j = tail.rfind(b"Code:", 0, i)
                text = tail[j if j >= 0 else i:].decode(errors="replace")
                m = re.search(r"Code:\s*(\d+)", text)
                raise ClickHouseError(int(m.group(1)) if m else -1, text)

    def count(self, sql: str) -> int:
        """The value of a ``SELECT count() ...`` (the rows hint of a streamed job)."""
        return int(self._post(sql.rstrip() + " FORMAT TabSeparated").strip() or 0)

    def insert_native(self, table: str, block: bytes) -> None:
        self._post("INSERT INTO %s FORMAT Native" % table, block)


def raw_select_sql(plan: QueryPlan, pod_label=None, pod_name=None, pod_namespace=None, ipv4_pushdown: bool = False) -> str:
    """The SELECT this job sends instead of generate_tad_sql_query's text: the raw ``flows`` columns the plan needs.
    Grouping, max / sum, the namespace ignore list and the string predicates run here (GPU / host), so ClickHouse only
    scans; the time window is still pushed down with the reference's own conditions (:581-586) to bound the transfer."""
    cols = ["flowEndSeconds", "throughput"]
    for br in plan.branches:
        for src in br.key.values():
            if isinstance(src, str) and src not in cols:
                cols.append(src)
    extra = []
    if plan.agg_flow == "pod":
        for side in ("source", "destination"):
            extra += [side + "PodLabels"] + ([side + "PodName"] if pod_name else []) + \
                     ([side + "PodNamespace"] if (pod_namespace and (pod_label or pod_name)) else [])
    elif plan.agg_flow == "external":
        extra += ["flowType", "destinationIP"]
    elif plan.agg_flow == "svc":
        extra += ["destinationServicePortName"]
    if plan.ns_ignore:
        extra += ["sourcePodNamespace", "destinationPodNamespace"]
    for c in extra:
        if c not in cols:
            cols.append(c)
    if ipv4_pushdown:
        # IPv4-only tables: let ClickHouse hand over the addresses as UInt32 (fixed width, copied without decoding) instead
        # of text -- text addresses cap the host-side ingest at ~1e7 rows/s per core.  IPv4StringToNum throws on anything
        # else, so a dual-stack table fails the query and the job is rerun in text mode.
        cols = ["IPv4StringToNum({0}) AS {0}".format(c) if c in ("sourceIP", "destinationIP") else c for c in cols]
    return "SELECT {} FROM {}".format(", ".join(cols), TABLE_NAME) + _window_where(plan)


def _window_where(plan: QueryPlan) -> str:
    where = []
    if plan.start_time:
        where.append("flowStartSeconds >= '{}'".format(plan.start_time))
    if plan.end_time:
        where.append("flowEndSeconds < '{}'".format(plan.end_time))
    return " WHERE " + " AND ".join(where) if where else ""


def count_sql(plan: QueryPlan) -> str:
    """``SELECT count()`` over the window :func:`raw_select_sql` reads: the rows of one streamed round, before the host
    predicates (an upper bound, which the engine accepts as a hint)."""
    return "SELECT count() FROM {}".format(TABLE_NAME) + _window_where(plan)


def _select_blocks(transport, sql: str):
    """Factory of one round of the SELECT's decoded Native blocks; every call issues the SELECT again."""
    from . import clickhouse_native as chn

    def blocks():
        if hasattr(transport, "select_native_stream"):
            decoded = chn.read_blocks_stream(transport.select_native_stream(sql))
        else:
            decoded = chn.read_blocks(transport.select_native(sql))
        for cols, _types, _rows in decoded:
            yield cols
    return blocks


def _run_streamed(engine, transport, a: dict, plan: QueryPlan, pushdown: bool, tad_id: str, device_text: bool = False,
                  device_ns: bool = False):
    """main()'s job on streamed input (TAD_STREAM_INPUT=1): (result SoA, plan, dictionaries).  ``device_text``
    (TAD_DEVICE_TEXT=1: True, text addresses only; TAD_DEVICE_TEXT=all: "all"): run_engine_stream's ``device_text``.
    ``device_ns`` (TAD_DEVICE_NS=1): run_engine_stream's ``device_ns``, with and without push-down."""
    hint = 0
    if hasattr(transport, "count"):
        hint = int(transport.count(count_sql(plan))) * len(plan.branches)    # pod: every row feeds both branches
    if os.getenv("TAD_HOST_BUDGET") is not None:
        engine.set_host_budget(int(os.getenv("TAD_HOST_BUDGET")))

    def run(ipv4_pushdown):
        sql = raw_select_sql(plan, a["pod_label"], a["pod_name"], a["pod_namespace"], ipv4_pushdown=ipv4_pushdown)
        return run_engine_stream(engine, a["algo"], _select_blocks(transport, sql), a["start_time"], a["end_time"], tad_id,
                                 a["ns_ignore_list"], a["agg_flow"] or None, a["pod_label"] or None, a["external_ip"] or None,
                                 a["svc_port_name"] or None, a["pod_name"] or None, a["pod_namespace"] or None, rows_hint=hint,
                                 device_text=False if ipv4_pushdown else device_text, device_ns=device_ns)
    try:
        got, _st, plan, dicts = run(pushdown)
    except Exception as e:
        if not pushdown or not _is_ipv4_pushdown_failure(e):
            raise
        # ClickHouse may reject a non-IPv4 address after some blocks were pushed: that job was cancelled and released
        logger.info("IPv4 push-down failed (non-IPv4 addresses?): rerunning the job with the addresses as text")
        got, _st, plan, dicts = run(False)
    return got, plan, dicts


def main(argv=None, engine=None, transport=None) -> int:
    """Drop-in for ``python anomaly_detection.py <argv>`` (anomaly_detection.py:729-900): reads ``default.flows``,
    writes ``default.tadetector``, logs the same completion line.  ``engine`` / ``transport`` are injection points for
    the tests; in the job container they are the GPU engine and the ClickHouse HTTP endpoint of ``--db_jdbc_url``."""
    from . import clickhouse_native as chn
    try:
        a = parse_args(sys.argv[1:] if argv is None else argv)
    except getopt.GetoptError:
        return 2                                                    # the reference exits 2 on bad options (:800-803)
    t0 = time.time()
    logger.info("Script started at {}".format(datetime.now().strftime("%a, %d %B %Y %H:%M:%S")))
    if a["algo"] not in VALID_ALGOS:
        raise ValueError("Algorithm should be in {}".format(" or ".join(VALID_ALGOS)))
    own_engine = engine is None
    if own_engine:
        from .engine import TadEngine
        engine = TadEngine(device=int(os.getenv("TAD_DEVICE", "0")))
    transport = transport or ClickHouseHTTP(a["db_jdbc_url"])
    try:
        plan = plan_query(a["start_time"], a["end_time"], a["ns_ignore_list"], a["agg_flow"], a["pod_label"], a["external_ip"],
                          a["svc_port_name"], a["pod_name"], a["pod_namespace"])
        pushdown = os.getenv("TAD_IPV4_PUSHDOWN", "0") == "1"
        if os.getenv("TAD_STREAM_INPUT", "0") == "1":       # blocks pushed to a streamed job as they are decoded
            tad_id = a["id"] or str(uuid.uuid4())
            # TAD_DEVICE_TEXT=1: the address text of a connection-mode job is dictionary-encoded on the GPU (no push-down);
            # TAD_DEVICE_TEXT=all: every mode's String keys, its string predicates evaluated on the GPU
            device_text = {"1": True, "all": "all"}.get(os.getenv("TAD_DEVICE_TEXT", "0"), False) if not pushdown else False
            # TAD_DEVICE_NS=1: the namespace ignore list is tested on the GPU from the namespace text columns
            device_ns = os.getenv("TAD_DEVICE_NS", "0") == "1"
            got, plan, dicts = _run_streamed(engine, transport, a, plan, pushdown, tad_id, device_text, device_ns)
        else:
            sql = raw_select_sql(plan, a["pod_label"], a["pod_name"], a["pod_namespace"], ipv4_pushdown=pushdown)
            def read(q):          # block-by-block while the response arrives when the transport can stream, else the whole body
                if hasattr(transport, "select_native_stream"):
                    return chn.flows_from_native(transport.select_native_stream(q))
                return chn.flows_from_native(transport.select_native(q))
            try:
                flows = read(sql)
            except Exception as e:
                if not pushdown or not _is_ipv4_pushdown_failure(e):
                    raise
                logger.info("IPv4 push-down failed (non-IPv4 addresses?): reading the addresses as text")
                sql = raw_select_sql(plan, a["pod_label"], a["pod_name"], a["pod_namespace"])
                flows = read(sql)
            for c in (x.split(" AS ")[-1] for x in sql[len("SELECT "):sql.index(" FROM ")].split(", ")):   # empty table: no block at all
                flows.setdefault(c, np.zeros(0, dtype=np.uint64 if c == "throughput" else np.uint32))
            tad_id = a["id"] or str(uuid.uuid4())                               # write_anomaly_detection_result (:715-718)
            got, _st, plan, dicts = run_engine(engine, a["algo"], flows, a["start_time"], a["end_time"], tad_id, a["ns_ignore_list"],
                                               a["agg_flow"] or None, a["pod_label"] or None, a["external_ip"] or None,
                                               a["svc_port_name"] or None, a["pod_name"] or None, a["pod_namespace"] or None)
        if len(got["flow_end"]):                                           # column-wise: no Python object per result row
            block = chn.tadetector_block_from_result(got, plan, dicts, a["algo"], tad_id)
        else:                                                               # the NO ANOMALY DETECTED sentinel (:395-420)
            block = chn.tadetector_block(_result_rows(got, plan, dicts, a["algo"], tad_id, a["pod_label"] or None))
        transport.insert_native(RESULT_TABLE_NAME, block)
    finally:
        if own_engine:
            engine.close()
    logger.info("Anomaly Detection completed, id: {}, in {} seconds ".format(tad_id, time.time() - t0))
    return 0


if __name__ == "__main__":
    logging.basicConfig(level=logging.INFO)
    sys.exit(main())
