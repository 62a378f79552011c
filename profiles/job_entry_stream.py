"""The job entry point (`python -m theia_b200.anomaly_detection`) one-shot and on streamed input (TAD_STREAM_INPUT=1,
DESIGN.md section 10): wall time of main() and the process's peak resident memory, over an in-process ClickHouse double
that serves a configs[1]-shaped `flows` table (1e8 rows / 1e6 connections x 100 points, EWMA, connection mode) as Native
blocks of 65,536 and of 8M rows.

    python profiles/job_entry_stream.py [--series 1000000] [--points 100] [--blocks 65536 8388608]

The double generates every block on request from the row index, so it holds no table: what a run keeps in memory is what
the job entry point keeps.  Addresses arrive as UInt32 (TAD_IPV4_PUSHDOWN=1), so no String column is decoded.  Each run is
a process of its own, because the peak RSS (``resource.getrusage``) is a per-process high-water mark; ``source`` runs
only read and decode the blocks, the baseline of the two job paths.  The result digest (sorted result columns) must be
the same for every run.  Prints one JSON line per run, the card and its power limit first; writes nothing."""
import argparse
import hashlib
import json
import os
import resource
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

SPIKES = np.array([0.1, 2.5, 12.0])
TYPES = {"flowEndSeconds": "DateTime", "throughput": "UInt64", "sourceTransportPort": "UInt16",
         "destinationTransportPort": "UInt16", "protocolIdentifier": "UInt8", "flowStartSeconds": "DateTime"}


def _mix(x):
    """splitmix64 finaliser: a per-row random word from the row index (uint64 arithmetic wraps)."""
    x = (x + np.uint64(0x9E3779B97F4A7C15))
    x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


class SynthTransport:
    """Row r of the table is point r // S + 1 of connection r % S; the connections' attributes come from a seeded rng,
    the throughput from a hash of r (noise of 1e-3 and 1 % spikes, as theia_b200.synth.make_flows)."""

    def __init__(self, series, points, block_rows, seed=1):
        from theia_b200 import synth
        rng = np.random.default_rng(seed)
        S = self.S = series
        self.rows, self.block_rows = series * points, block_rows
        self.src_ip = (np.uint32(10 << 24) + rng.integers(0, 1 << 24, S, dtype=np.uint32)).astype(np.uint32)
        self.dst_ip = (np.uint32(10 << 24) + rng.integers(0, 1 << 24, S, dtype=np.uint32)).astype(np.uint32)
        self.src_port = rng.integers(1024, 65536, S).astype(np.uint16)
        self.dst_port = synth.SERVICE_PORTS[rng.integers(0, len(synth.SERVICE_PORTS), S)]
        self.proto = np.where(rng.random(S) < 0.8, 6, 17).astype(np.uint8)
        self.flow_start = (synth.T0 + rng.integers(0, 3600, S)).astype(np.uint32)
        self.base = np.exp(rng.uniform(np.log(1e6), np.log(1e10), S))
        self.selects, self.body = 0, None

    def _block(self, lo, hi):
        r = np.arange(lo, hi, dtype=np.uint64)
        sid = (r % np.uint64(self.S)).astype(np.int64)
        k = (r // np.uint64(self.S)).astype(np.int64) + 1
        h = _mix(r)
        u = (h >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
        val = self.base[sid] * (1.0 + 2e-3 * (u - 0.5))
        val = np.where((h & np.uint64(127)) == 0, val * SPIKES[(h >> np.uint64(7)) % np.uint64(3)], val)
        return {"sourceIP": self.src_ip[sid], "destinationIP": self.dst_ip[sid], "sourceTransportPort": self.src_port[sid],
                "destinationTransportPort": self.dst_port[sid], "protocolIdentifier": self.proto[sid],
                "flowStartSeconds": self.flow_start[sid], "flowEndSeconds": (self.flow_start[sid] + 60 * k).astype(np.uint32),
                "throughput": np.maximum(np.rint(val), 1.0).astype(np.uint64)}

    def count(self, sql):
        return self.rows

    def select_native_stream(self, sql):
        from theia_b200 import clickhouse_native as chn
        self.selects += 1
        spec = []
        for x in sql[len("SELECT "):sql.index(" FROM ")].split(", "):
            name = x.split(" AS ")[-1]
            assert x.startswith("IPv4StringToNum(") or name in TYPES, x
            spec.append((name, TYPES.get(name, "UInt32")))
        for lo in range(0, self.rows, self.block_rows):
            b = self._block(lo, min(self.rows, lo + self.block_rows))
            yield chn.write_native([(name, typ, b[name]) for name, typ in spec])

    def insert_native(self, table, body):
        self.body = body


def _digest(body) -> str:
    from theia_b200 import clickhouse_native as chn
    h = hashlib.sha256()
    for cols, _types, _rows in chn.read_blocks(body):
        for name in ("sourceTransportPort", "destinationTransportPort", "flowStartSeconds", "flowEndSeconds",
                     "throughputStandardDeviation", "algoCalc", "throughput"):
            h.update(np.sort(np.asarray(cols[name])).tobytes())
    return h.hexdigest()[:16]


def run_one(path, series, points, block_rows):
    os.environ["TAD_IPV4_PUSHDOWN"] = "1"
    from theia_b200 import anomaly_detection as ad
    from theia_b200 import clickhouse_native as chn
    tr = SynthTransport(series, points, block_rows)
    rss0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    out = {"path": path, "block_rows": block_rows, "rows": tr.rows}
    t0 = time.perf_counter()
    if path == "source":
        sql = ad.raw_select_sql(ad.plan_query(), ipv4_pushdown=True)
        out["blocks"] = sum(1 for _ in chn.read_blocks_stream(tr.select_native_stream(sql)))
    else:
        from theia_b200.engine import TadEngine
        os.environ["TAD_STREAM_INPUT"] = "1" if path == "streamed" else "0"
        with TadEngine(device=0) as eng:
            eng.run({"flow_end": np.zeros(1, np.uint32), "value": np.ones(1, np.uint64)})     # context warm-up
            rss0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
            t0 = time.perf_counter()
            assert ad.main(["--algo", "EWMA", "--id", "profile"], engine=eng, transport=tr) == 0
            out["wall_s"] = time.perf_counter() - t0
            peak = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
        out["selects"] = tr.selects
        out["result_digest"] = _digest(tr.body)
    if path == "source":
        peak = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    wall = time.perf_counter() - t0 if path == "source" else out["wall_s"]
    out["wall_s"] = round(wall, 2)
    out["records_per_s"] = float("%.3g" % (tr.rows / wall))
    out["rss_before_mb"] = round(rss0 / 1024)
    out["peak_rss_mb"] = round(peak / 1024)          # ru_maxrss: KiB on Linux
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1_000_000)
    ap.add_argument("--points", type=int, default=100)
    ap.add_argument("--blocks", type=int, nargs="+", default=[65536, 8 << 20])
    ap.add_argument("--paths", nargs="+", default=["source", "one-shot", "streamed"])
    ap.add_argument("--run", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.run:
        run_one(args.run, args.series, args.points, args.blocks[0])
        return
    from profiles.memory_budget import card
    print(json.dumps(card()), flush=True)
    for block in args.blocks:
        for path in args.paths:
            subprocess.run([sys.executable, os.path.abspath(__file__), "--run", path, "--series", str(args.series),
                            "--points", str(args.points), "--blocks", str(block)], check=True)


if __name__ == "__main__":
    main()
