"""The job entry point with a namespace ignore list on streamed input (DESIGN.md section 10, "The namespace ignore list on
the device"): wall time of main(), records/s and peak resident memory over an in-process ClickHouse double that serves a
configs[1]-shaped `flows` table (connection id = row % S, EWMA) as Native blocks, with 40 namespaces per side and an
ignore list of 3 names (two of them present).

    python profiles/job_entry_ns.py [--series 100000] [--points 100] [--blocks 65536 8388608] [--variants text pushdown]

Variants (connection mode): text -- the addresses as IPv4 text, dictionary-encoded on the GPU (TAD_DEVICE_TEXT=1);
pushdown -- the addresses as UInt32 (TAD_IPV4_PUSHDOWN=1).  Paths, each a process of its own (peak RSS is a per-process
high-water mark):
  source      generate + decode the blocks only
  host-ns     TAD_STREAM_INPUT=1: the namespace columns are dictionary-encoded on the host, the list goes as ids
  device-ns   TAD_STREAM_INPUT=1 TAD_DEVICE_NS=1: the namespace columns go as text, the list as names, tested on the GPU
The result digest must be the same for both engine paths of a variant.  Prints one JSON line per run, the card and its
power limit first; writes nothing."""
import argparse
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

from profiles.job_entry_modes import FIXED, ModesTransport, digest  # noqa: E402
from profiles.job_entry_text import _Status  # noqa: E402

IGNORE = ["namespace-03", "namespace-17", "kube-system"]


class NsTransport(ModesTransport):
    """ModesTransport with the connection mode's address columns: IPv4 text, or UInt32 under IPv4StringToNum."""

    def __init__(self, series, points, block_rows, seed=1):
        super().__init__(series, points, block_rows, seed)
        from theia_b200 import anomaly_detection as ad
        from theia_b200 import clickhouse_native as chn
        enc = np.empty(self.S, dtype=object)
        enc[:] = [chn._enc_string(ad.u32_to_ip(int(v))) for v in self.src_ip]
        self.enc["sourceIP"] = enc

    def select_native_stream(self, sql):
        from theia_b200 import clickhouse_native as chn
        self.selects += 1
        spec = []
        for x in sql[len("SELECT "):sql.index(" FROM ")].split(", "):
            name = x.split(" AS ")[-1]
            spec.append((name, "UInt32" if x.startswith("IPv4StringToNum(") else FIXED.get(name, "String")))
        for lo in range(0, self.rows, self.block_rows):
            hi = min(self.rows, lo + self.block_rows)
            b = self._block(lo, hi)
            sid = (np.arange(lo, hi, dtype=np.uint64) % np.uint64(self.S)).astype(np.int64)
            out = [chn._enc_varuint(len(spec)), chn._enc_varuint(hi - lo)]
            for name, typ in spec:
                out += [chn._enc_string(name), chn._enc_string(typ)]
                if typ == "String":
                    out.append(b"".join(self.enc[name][sid].tolist()))
                else:
                    out.append(np.ascontiguousarray(b[name], dtype=chn._FIXED[typ]).tobytes())
            yield b"".join(out)


def run_one(path, variant, series, points, block_rows):
    os.environ["TAD_STREAM_INPUT"] = "1"
    os.environ["TAD_IPV4_PUSHDOWN"] = "1" if variant == "pushdown" else "0"
    os.environ["TAD_DEVICE_TEXT"] = "1" if variant == "text" else "0"
    os.environ["TAD_DEVICE_NS"] = "1" if path == "device-ns" else "0"
    from theia_b200 import anomaly_detection as ad
    from theia_b200 import clickhouse_native as chn
    tr = NsTransport(series, points, block_rows)
    argv = ["--algo", "EWMA", "--id", "profile", "--ns-ignore-list", json.dumps(IGNORE)]
    out = {"variant": variant, "path": path, "block_rows": block_rows, "rows": tr.rows}
    rss0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    if path == "source":
        t0 = time.perf_counter()
        plan = ad.plan_query(ns_ignore_list=IGNORE)
        sql = ad.raw_select_sql(plan, ipv4_pushdown=variant == "pushdown")
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
            assert ad.main(argv, engine=eng, transport=tr) == 0
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
    ap.add_argument("--variants", nargs="+", default=["text", "pushdown"])
    ap.add_argument("--paths", nargs="+", default=["source", "host-ns", "device-ns"])
    ap.add_argument("--run", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.run:
        path, variant = args.run.split(":")
        run_one(path, variant, args.series, args.points, args.blocks[0])
        return
    from profiles.memory_budget import card
    print(json.dumps(card()), flush=True)
    for variant in args.variants:
        for block in args.blocks:
            for path in args.paths:
                subprocess.run([sys.executable, os.path.abspath(__file__), "--run", "%s:%s" % (path, variant), "--series",
                                str(args.series), "--points", str(args.points), "--blocks", str(block)], check=True)


if __name__ == "__main__":
    main()
