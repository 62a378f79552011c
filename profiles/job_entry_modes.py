"""The job entry point's aggregated-flow modes on streamed input (DESIGN.md section 10, "String predicates on the device"):
wall time of main(), records/s and peak resident memory over an in-process ClickHouse double that serves a
configs[1]-shaped `flows` table (connection id = row % S, EWMA) as Native blocks with the String columns of the
external, pod and svc modes.

    python profiles/job_entry_modes.py [--series 100000] [--points 100] [--blocks 65536 8388608] [--modes external pod svc]

Modes: external (one destinationIP per connection, so about as many external IPs as connections; flowType 1, 2 or 3 per
connection), pod with --pod-label app (JSON labels of 60-90 bytes, longer than the text staging's 48 bytes per row,
half of them with an "app" key; 40 namespaces), svc (500 service port names and one connection in ten without one).
Paths, each a process of its own (peak RSS is a per-process high-water mark):
  source         generate + decode the blocks only
  host-dict      TAD_STREAM_INPUT=1: the host applies the string predicates and codes every block's String keys
  device-text    TAD_STREAM_INPUT=1 TAD_DEVICE_TEXT=all: String keys as text, the predicates evaluated on the GPU
The result digest (sorted numeric result columns and sorted names) must be the same for every path of a mode.  Prints one
JSON line per run, the card and its power limit first; writes nothing."""
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

from profiles.job_entry_stream import TYPES, SynthTransport, _digest  # noqa: E402
from profiles.job_entry_text import _Status  # noqa: E402

MODE_ARGS = {"external": ["--agg-flow", "external"], "pod": ["--agg-flow", "pod", "--pod-label", "app"],
             "svc": ["--agg-flow", "svc"]}
NAME_COLS = ("destinationIP", "destinationServicePortName", "podNamespace", "podLabels", "podName")
FIXED = dict(TYPES, flowType="UInt8")


class ModesTransport(SynthTransport):
    """SynthTransport with the String columns of the aggregated-flow modes, one value per connection."""

    def __init__(self, series, points, block_rows, seed=1):
        super().__init__(series, points, block_rows, seed)
        from theia_b200 import anomaly_detection as ad
        from theia_b200 import clickhouse_native as chn
        rng = np.random.default_rng(seed + 1)
        S = self.S
        self.flow_type = rng.choice(np.array([1, 2, 3], dtype=np.uint8), S)
        ns = ["namespace-%02d" % k for k in range(40)]
        labels = []
        for k in range(4000):
            d = {"pod-template-hash": "%010x" % (k * 2654435761 % (1 << 40)), "tier": "t%d" % (k % 7),
                 "team": "team-%03d" % (k % 300)}
            if k % 2:
                d["app"] = "service-%04d" % k
            labels.append(json.dumps(d, sort_keys=True))
        svc = [""] + ["namespace-%02d/svc-%03d:port-%d" % (k % 40, k, k % 3) for k in range(500)]
        per_series = {
            "destinationIP": [ad.u32_to_ip(int(v)) for v in self.dst_ip],
            "sourcePodNamespace": [ns[k] for k in rng.integers(0, len(ns), S)],
            "destinationPodNamespace": [ns[k] for k in rng.integers(0, len(ns), S)],
            "sourcePodLabels": [labels[k] for k in rng.integers(0, len(labels), S)],
            "destinationPodLabels": [labels[k] for k in rng.integers(0, len(labels), S)],
            "destinationServicePortName": [svc[0] if k % 10 == 0 else svc[1 + k % 500] for k in rng.integers(0, 10**6, S)],
        }
        self.enc = {}
        for name, text in per_series.items():
            enc = np.empty(S, dtype=object)
            enc[:] = [chn._enc_string(s) for s in text]
            self.enc[name] = enc

    def select_native_stream(self, sql):
        from theia_b200 import clickhouse_native as chn
        self.selects += 1
        spec = []
        for x in sql[len("SELECT "):sql.index(" FROM ")].split(", "):
            name = x.split(" AS ")[-1]
            spec.append((name, FIXED.get(name, "String")))
        for lo in range(0, self.rows, self.block_rows):
            hi = min(self.rows, lo + self.block_rows)
            b = self._block(lo, hi)
            sid = (np.arange(lo, hi, dtype=np.uint64) % np.uint64(self.S)).astype(np.int64)
            b["flowType"] = self.flow_type[sid]
            out = [chn._enc_varuint(len(spec)), chn._enc_varuint(hi - lo)]
            for name, typ in spec:
                out += [chn._enc_string(name), chn._enc_string(typ)]
                if typ == "String":
                    out.append(b"".join(self.enc[name][sid].tolist()))
                else:
                    out.append(np.ascontiguousarray(b[name], dtype=chn._FIXED[typ]).tobytes())
            yield b"".join(out)


def digest(body) -> str:
    """_digest's numeric columns, then every name column sorted."""
    from theia_b200 import clickhouse_native as chn
    h = hashlib.sha256(_digest(body).encode())
    for cols, _types, _rows in chn.read_blocks(body):
        for name in NAME_COLS:
            if name in cols:
                c = cols[name]
                vals = [str(x) for x in (c.to_list() if hasattr(c, "to_list") else c)]
                h.update("\n".join(sorted(vals)).encode())
    return h.hexdigest()[:16]


def run_one(path, mode, series, points, block_rows):
    os.environ["TAD_STREAM_INPUT"] = "1"
    os.environ["TAD_IPV4_PUSHDOWN"] = "0"
    os.environ["TAD_DEVICE_TEXT"] = "all" if path == "device-text" else "0"
    from theia_b200 import anomaly_detection as ad
    from theia_b200 import clickhouse_native as chn
    tr = ModesTransport(series, points, block_rows)
    argv = MODE_ARGS[mode]
    out = {"mode": mode, "path": path, "block_rows": block_rows, "rows": tr.rows}
    rss0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    if path == "source":
        t0 = time.perf_counter()
        a = ad.parse_args(["--algo", "EWMA"] + argv)
        plan = ad.plan_query(a["start_time"], a["end_time"], a["ns_ignore_list"], a["agg_flow"], a["pod_label"])
        sql = ad.raw_select_sql(plan, a["pod_label"], a["pod_name"], a["pod_namespace"])
        out["blocks"] = sum(1 for _ in chn.read_blocks_stream(tr.select_native_stream(sql)))
        wall = time.perf_counter() - t0
    else:
        from theia_b200.engine import TadEngine
        e = TadEngine(device=0)
        try:
            e.run({"flow_end": np.zeros(1, np.uint32), "value": np.ones(1, np.uint64)})     # context warm-up
            eng = _Status(e)
            rss0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
            t0 = time.perf_counter()
            assert ad.main(["--algo", "EWMA", "--id", "profile"] + argv, engine=eng, transport=tr) == 0
            wall = time.perf_counter() - t0
        finally:
            e.close()
        st = eng.status[-1]
        out["rows_kept"] = st["rows_kept"]
        out["device_ms"] = round(st["device_ms"], 1)
        out["selects"] = tr.selects
        out["result_digest"] = digest(tr.body)
    out["wall_s"] = round(wall, 2)
    out["records_per_s"] = float("%.3g" % (tr.rows / wall))
    out["rss_before_mb"] = round(rss0 / 1024)
    out["peak_rss_mb"] = round(resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024)    # ru_maxrss: KiB on Linux
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=100_000)
    ap.add_argument("--points", type=int, default=100)
    ap.add_argument("--blocks", type=int, nargs="+", default=[65536, 8 << 20])
    ap.add_argument("--modes", nargs="+", default=["external", "pod", "svc"])
    ap.add_argument("--paths", nargs="+", default=["source", "host-dict", "device-text"])
    ap.add_argument("--run", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.run:
        path, mode = args.run.split(":")
        run_one(path, mode, args.series, args.points, args.blocks[0])
        return
    from profiles.memory_budget import card
    print(json.dumps(card()), flush=True)
    for mode in args.modes:
        for block in args.blocks:
            for path in args.paths:
                subprocess.run([sys.executable, os.path.abspath(__file__), "--run", "%s:%s" % (path, mode), "--series",
                                str(args.series), "--points", str(args.points), "--blocks", str(block)], check=True)


if __name__ == "__main__":
    main()
