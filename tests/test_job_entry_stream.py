"""The job entry point on streamed input (TAD_STREAM_INPUT=1): main() pushes every decoded Native block of its SELECT to a
streamed engine job instead of concatenating the blocks into one table.  The INSERT body must equal the one of the default
path on the same ClickHouse data, in every aggregation mode."""
import json
import re
from datetime import datetime

import numpy as np
import pytest

from theia_b200 import anomaly_detection as ad
from theia_b200 import clickhouse_native as chn
from theia_b200 import synth

from .test_host_mirror_on_oracle import OracleEngine

TYPES = {"sourceIP": "String", "destinationIP": "String", "sourceTransportPort": "UInt16",
         "destinationTransportPort": "UInt16", "protocolIdentifier": "UInt8", "flowStartSeconds": "DateTime",
         "flowEndSeconds": "DateTime", "throughput": "UInt64", "flowType": "UInt8"}     # every other column: String
BLOCK_ROWS = 3000


def make_table(series=300, points=40, seed=11, dual_stack=False, block_rows=BLOCK_ROWS):
    """A seeded ``flows`` table (theia_b200.synth) with the String columns of every aggregation mode.  ``dual_stack``: the
    source addresses are text, some of them IPv6, none in the first block (so a push-down SELECT fails mid-stream)."""
    t = synth.make_flows(series, points, seed=seed)
    n = len(t["value"])
    rng = np.random.default_rng(seed)
    pods = t["src_ip"] % 17
    dpods = t["dst_ip"] % 13
    ns = np.array(["default", "kube-system", "shop", "flow-visibility"], dtype=object)
    labels = np.array(['{"app":"web","pod-template-hash":"%d"}' % i if i % 3 else "" for i in range(17)], dtype=object)
    svc = np.array(["", "shop/web:http", "shop/db:pg", "default/dns:udp"], dtype=object)
    fl = {"sourceIP": t["src_ip"], "destinationIP": t["dst_ip"], "sourceTransportPort": t["src_port"],
          "destinationTransportPort": t["dst_port"], "protocolIdentifier": t["proto"], "flowStartSeconds": t["flow_start"],
          "flowEndSeconds": t["flow_end"], "throughput": t["value"],
          "flowType": rng.choice(np.array([1, 2, 3], dtype=np.uint8), n),
          "sourcePodNamespace": ns[pods % 4], "destinationPodNamespace": ns[dpods % 4],
          "sourcePodLabels": labels[pods], "destinationPodLabels": labels[dpods],
          "sourcePodName": np.array(["pod-%d" % p for p in pods], dtype=object),
          "destinationPodName": np.array(["pod-%d" % p for p in dpods], dtype=object),
          "destinationServicePortName": svc[dpods % 4]}
    if dual_stack:
        src = np.array([ad.u32_to_ip(int(v)) for v in t["src_ip"]], dtype=object)
        v6 = (t["src_ip"] % 5 == 0) & (np.arange(n) >= block_rows)
        src[v6] = ["fd00::%x" % int(v) for v in t["src_ip"][v6]]
        fl["sourceIP"] = src
    return fl


class TableTransport:
    """ClickHouse double over a flows table: answers raw_select_sql's SELECT with the named columns of the rows in its
    time window, as Native blocks of ``block_rows`` rows through select_native_stream (IPv4StringToNum columns as UInt32;
    a non-IPv4 value fails the stream with ClickHouse's trailer once the blocks before it are sent), and count()."""

    def __init__(self, flows, block_rows=BLOCK_ROWS, events=None):
        self.flows, self.block_rows = flows, block_rows
        self.events = [] if events is None else events
        self.selects, self.counts, self.inserts = [], [], []

    def _rows(self, sql):
        keep = np.ones(len(self.flows["flowEndSeconds"]), dtype=bool)
        for col, op, ts in re.findall(r"(flowStartSeconds|flowEndSeconds) (>=|<) '([^']+)'", sql):
            v = np.asarray(self.flows[col]).astype(np.int64)
            keep &= (v >= ad._epoch(ts)) if op == ">=" else (v < ad._epoch(ts))
        return np.flatnonzero(keep)

    def count(self, sql):
        assert sql.startswith("SELECT count() FROM default.flows")
        self.counts.append(sql)
        return len(self._rows(sql))

    def select_native_stream(self, sql):
        self.selects.append(sql)
        return self._pieces(sql)

    def _pieces(self, sql):
        rows = self._rows(sql)
        spec = []
        for x in sql[len("SELECT "):sql.index(" FROM ")].split(", "):
            name = x.split(" AS ")[-1]
            spec.append((name, "UInt32" if x.startswith("IPv4StringToNum(") else TYPES.get(name, "String")))
        for b, lo in enumerate(range(0, len(rows), self.block_rows)):
            sel = rows[lo:lo + self.block_rows]
            cols = []
            for name, typ in spec:
                v = np.asarray(self.flows[name])[sel]
                if typ == "UInt32" and v.dtype.kind not in "iu":
                    try:
                        v = ad.ip_to_u32(v)
                    except ValueError:
                        raise ad.ClickHouseError(441, "Code: 441. DB::Exception: Cannot parse IPv4 from String")
                elif typ == "String" and v.dtype.kind in "iu":
                    v = v.astype(np.uint32)                     # an IPv4 key column: written as dotted quads
                cols.append((name, typ, v))
            self.events.append(("block", b))
            yield chn.write_native(cols)

    def insert_native(self, table, block):
        self.inserts.append((table, block))


class StreamJob:
    def __init__(self, eng, kw):
        self.eng, self.kw = eng, kw
        self.pushes, self.rounds = [[]], 0
        self.cancelled = self.released = False

    def push(self, block):
        assert not self.released
        self.pushes[-1].append({k: (None if v is None else np.array(v)) for k, v in block.items()})
        self.eng.events.append(("push", len(block["flow_end"])))

    def end(self):
        self.rounds += 1
        again = self.rounds < self.eng.rounds
        if again:
            self.pushes.append([])
        return again

    def wait(self):
        kw, first = self.kw, self.pushes[0]
        table = {"flow_end": np.zeros(0, np.uint32), "value": np.zeros(0, np.uint64)}
        if first:
            table = {k: (None if any(p[k] is None for p in first) else np.concatenate([p[k] for p in first]))
                     for k in first[0]}
        self.got, st = OracleEngine()._run(table, kw["algo"], kw["reducer"], kw["start_time"], kw["end_time"], kw["ns_ignore"])
        return st

    def result(self):
        return self.got

    def cancel(self):
        self.cancelled = True

    def release(self):
        self.released = True


class StreamEngine:
    """Stands in for TadEngine's streamed jobs: records every job's pushes per round, asks for ``rounds`` rounds and
    answers with the CPU oracle over the first round's rows."""

    def __init__(self, rounds=1, events=None):
        self.rounds, self.jobs, self.host_budget = rounds, [], None
        self.events = [] if events is None else events

    def submit_stream(self, **kw):
        self.jobs.append(StreamJob(self, kw))
        return self.jobs[-1]

    def set_host_budget(self, nbytes):
        self.host_budget = nbytes


class _FixedNow(datetime):
    @classmethod
    def now(cls, tz=None):
        return datetime(2026, 1, 2, 3, 4, 5)


@pytest.fixture(autouse=True)
def fixed_clock(monkeypatch):
    """The sentinel row carries the time of the job; both paths must see the same one."""
    monkeypatch.setattr(ad, "datetime", _FixedNow)


def canonical_rows(body):
    got = chn.read_native(body)
    cols = sorted(got)
    return sorted(tuple(str(got[c][i]) for c in cols) for i in range(len(got["id"])))


def both_paths(monkeypatch, argv, flows, rounds=1):
    """(default-path rows, streamed rows, transport, engine) of one argv over the same data."""
    monkeypatch.delenv("TAD_STREAM_INPUT", raising=False)
    tr = TableTransport(flows)
    assert ad.main(argv, engine=OracleEngine(), transport=tr) == 0
    want = canonical_rows(tr.inserts[0][1])
    monkeypatch.setenv("TAD_STREAM_INPUT", "1")
    eng, tr2 = StreamEngine(rounds), TableTransport(flows)
    assert ad.main(argv, engine=eng, transport=tr2) == 0
    (name, body), = tr2.inserts
    assert name == "default.tadetector"
    return want, canonical_rows(body), tr2, eng


WINDOW = ["--start_time", "2022-08-11 06:40:00", "--end_time", "2022-08-11 07:40:00"]
MODES = {
    "connection-text": ([], False, False),
    "connection-pushdown": ([], True, False),
    "connection-dual-stack": ([], False, True),
    "connection-window": (WINDOW, False, False),
    "ns-ignore": (["--ns-ignore-list", '["kube-system", "no-such-ns"]'], False, False),
    "pod-label-namespace": (["--agg-flow", "pod", "--pod-label", "web", "--pod-namespace", "shop"], False, False),
    "pod-name-namespace": (["--agg-flow", "pod", "--pod-name", "pod-5", "--pod-namespace", "kube-system"], False, False),
    "pod-labels-ns-ignore": (["--agg-flow", "pod", "--ns-ignore-list", '["default"]'], False, False),
    "external": (["--agg-flow", "external"] + WINDOW, False, False),
    "external-ip": (["--agg-flow", "external", "--external-ip", None], False, False),
    "svc": (["--agg-flow", "svc"], False, False),
    "svc-port-name": (["--agg-flow", "svc", "--svc-port-name", "shop/web:http"], False, False),
}


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("algo", ["EWMA", "DBSCAN"])
def test_streamed_insert_body_equals_the_default_path(monkeypatch, mode, algo):
    extra, pushdown, dual = MODES[mode]
    flows = make_table(dual_stack=dual)
    extra = [ad.u32_to_ip(int(flows["destinationIP"][7])) if x is None else x for x in extra]
    if pushdown:
        monkeypatch.setenv("TAD_IPV4_PUSHDOWN", "1")
    want, got, tr, eng = both_paths(monkeypatch, ["--algo", algo, "--id", "s-" + mode] + extra, flows)
    assert got == want
    if mode.startswith("connection"):
        assert len(want) > 1, "no anomaly: the comparison would only see the sentinel row"
    (job,) = eng.jobs
    assert job.rounds == 1 and job.released and not job.cancelled
    assert len(tr.selects) == 1 and ("IPv4StringToNum" in tr.selects[0]) == pushdown
    pod = "--agg-flow" in extra and extra[extra.index("--agg-flow") + 1] == "pod"
    kept = sum(len(p["flow_end"]) for p in job.pushes[0])
    assert job.kw["rows_hint"] == len(tr._rows(tr.selects[0])) * (2 if pod else 1) >= kept
    if "--ns-ignore-list" in extra:
        assert len(job.kw["ns_ignore"]) == len(json.loads(extra[extra.index("--ns-ignore-list") + 1]))


def test_empty_table_writes_the_sentinel_row(monkeypatch):
    flows = {k: v[:0] for k, v in make_table().items()}
    want, got, _tr, eng = both_paths(monkeypatch, ["--algo", "EWMA", "--id", "empty", "--agg-flow", "svc"], flows)
    assert got == want and len(got) == 1 and "NO ANOMALY DETECTED" in got[0]
    assert eng.jobs[0].pushes == [[]]


def test_text_addresses_go_through_the_dictionary_and_keep_their_ids(monkeypatch):
    flows = make_table()
    monkeypatch.setenv("TAD_STREAM_INPUT", "1")
    eng, tr = StreamEngine(), TableTransport(flows)
    assert ad.main(["--algo", "EWMA", "--id", "d"], engine=eng, transport=tr) == 0
    src = np.concatenate([p["src_ip"] for p in eng.jobs[0].pushes[0]])
    addr = np.asarray(flows["sourceIP"]).astype(np.int64)       # every row is pushed, in order (no host predicate)
    distinct = len(np.unique(addr))
    # one id per address and one address per id: groups exactly as the text does
    assert len(np.unique(src)) == distinct == np.unique(np.stack([src.astype(np.int64), addr]), axis=1).shape[1]
    assert src.max() == distinct - 1                             # dense dictionary ids, not u32 addresses


def test_pushes_interleave_with_the_reads_and_stay_block_sized(monkeypatch):
    monkeypatch.setenv("TAD_STREAM_INPUT", "1")
    for extra, per_block in (([], 1), (["--agg-flow", "pod"], 2)):
        events = []
        flows = make_table()
        eng, tr = StreamEngine(events=events), TableTransport(flows, events=events)
        assert ad.main(["--algo", "EWMA", "--id", "i"] + extra, engine=eng, transport=tr) == 0
        blocks = [i for i, e in enumerate(events) if e[0] == "block"]
        pushes = [i for i, e in enumerate(events) if e[0] == "push"]
        assert len(blocks) == -(-len(flows["flowEndSeconds"]) // BLOCK_ROWS) > 2
        assert pushes[0] < blocks[-1] and pushes[0] < blocks[1]          # the first block is pushed before the second is read
        assert max(e[1] for e in events if e[0] == "push") <= BLOCK_ROWS
        assert len(pushes) <= per_block * len(blocks)
        assert len(eng.jobs[0].pushes[0]) == len(pushes)


def test_each_round_reissues_the_select_with_identical_ids(monkeypatch):
    monkeypatch.setenv("TAD_STREAM_INPUT", "1")
    for extra in ([], ["--agg-flow", "pod", "--ns-ignore-list", '["default"]']):
        flows = make_table(dual_stack=not extra)
        eng, tr = StreamEngine(rounds=2), TableTransport(flows)
        assert ad.main(["--algo", "EWMA", "--id", "r"] + extra, engine=eng, transport=tr) == 0
        assert len(tr.selects) == 2 and tr.selects[0] == tr.selects[1] and len(tr.counts) == 1
        first, second = eng.jobs[0].pushes
        assert len(first) == len(second) > 0
        for a, b in zip(first, second):
            assert a.keys() == b.keys()
            for k in a:
                assert (a[k] is None and b[k] is None) or np.array_equal(a[k], b[k]), k
    # and the body is the one of the default path
    want, got, tr, _eng = both_paths(monkeypatch, ["--algo", "EWMA", "--id", "r2"], make_table(), rounds=2)
    assert got == want and len(tr.selects) == 2


def test_pushdown_failure_mid_stream_cancels_and_reruns_in_text_mode(monkeypatch):
    flows = make_table(dual_stack=True)
    argv = ["--algo", "EWMA", "--id", "p"]
    want_text, got_text, _tr, _eng = both_paths(monkeypatch, argv, flows)
    assert got_text == want_text and len(want_text) > 1
    monkeypatch.setenv("TAD_IPV4_PUSHDOWN", "1")
    monkeypatch.setenv("TAD_STREAM_INPUT", "1")
    eng, tr = StreamEngine(), TableTransport(flows)
    assert ad.main(argv, engine=eng, transport=tr) == 0
    first, rerun = eng.jobs
    assert len(first.pushes[0]) >= 1 and first.cancelled and first.released and first.rounds == 0
    assert rerun.released and not rerun.cancelled and rerun.rounds == 1
    assert ["IPv4StringToNum" in q for q in tr.selects] == [True, False]
    assert canonical_rows(tr.inserts[0][1]) == got_text


def test_other_failures_are_not_retried(monkeypatch):
    monkeypatch.setenv("TAD_IPV4_PUSHDOWN", "1")
    monkeypatch.setenv("TAD_STREAM_INPUT", "1")

    class Broken(TableTransport):
        def _pieces(self, sql):
            yield from list(super()._pieces(sql))[:1]
            raise ad.ClickHouseError(241, "Code: 241. DB::Exception: Memory limit (total) exceeded")

    eng, tr = StreamEngine(), Broken(make_table())
    with pytest.raises(ad.ClickHouseError):
        ad.main(["--algo", "EWMA", "--id", "b"], engine=eng, transport=tr)
    (job,) = eng.jobs
    assert job.cancelled and job.released and len(tr.selects) == 1 and not tr.inserts


def test_hint_and_host_budget(monkeypatch):
    monkeypatch.setenv("TAD_STREAM_INPUT", "1")
    flows = make_table()

    class NoCount:                                       # a transport without count(): no hint
        def __init__(self):
            self.inner = TableTransport(flows)
            self.select_native_stream, self.insert_native = self.inner.select_native_stream, self.inner.insert_native

    eng = StreamEngine()
    assert ad.main(["--algo", "EWMA", "--id", "h"] + WINDOW, engine=eng, transport=NoCount()) == 0
    assert eng.jobs[0].kw["rows_hint"] == 0 and eng.host_budget is None
    monkeypatch.setenv("TAD_HOST_BUDGET", str(1 << 30))
    eng, tr = StreamEngine(), TableTransport(flows)
    assert ad.main(["--algo", "EWMA", "--id", "h"] + WINDOW, engine=eng, transport=tr) == 0
    assert eng.host_budget == 1 << 30
    assert tr.counts == ["SELECT count() FROM default.flows WHERE flowStartSeconds >= '2022-08-11 06:40:00' "
                         "AND flowEndSeconds < '2022-08-11 07:40:00'"]
    assert eng.jobs[0].kw["rows_hint"] == len(tr._rows(tr.counts[0])) < len(flows["flowEndSeconds"])


def test_run_engine_stream_rejects_an_unknown_algorithm():
    with pytest.raises(ValueError):
        ad.run_engine_stream(StreamEngine(), "KMEANS", lambda: iter(()))
