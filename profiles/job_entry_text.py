"""The job entry point on streamed input with text addresses (DESIGN.md section 10, "Text keys on the device"): wall time of
main(), records/s, peak resident memory and the h2d share of the job's device time, over an in-process ClickHouse double
that serves a configs[1]-shaped `flows` table (connection id = row % S, EWMA, connection mode) as Native blocks whose
sourceIP / destinationIP are String columns.

    python profiles/job_entry_text.py [--series 100000] [--points 100] [--blocks 65536 8388608] [--variants ipv4 ipv6]

Variants: every address IPv4 text, or one connection in five with `fd00::` IPv6 text.  Paths, each a process of its own
(peak RSS is a per-process high-water mark):
  source         generate + decode the blocks only
  host-dict      TAD_STREAM_INPUT=1: the host dictionary codes every block's address text
  device-text    TAD_STREAM_INPUT=1 TAD_DEVICE_TEXT=1: the address text is dictionary-encoded on the GPU
  pushdown       TAD_STREAM_INPUT=1 TAD_IPV4_PUSHDOWN=1 (IPv4 variant only): UInt32 addresses, the floor
The result digest (sorted numeric result columns) must be the same for every run of a variant.  Prints one JSON line
per run, the card and its power limit first; writes nothing."""
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

from profiles.job_entry_stream import TYPES, SynthTransport, _digest  # noqa: E402


class TextTransport(SynthTransport):
    """SynthTransport with the addresses as String columns unless the SELECT asks for IPv4StringToNum."""

    def __init__(self, series, points, block_rows, ipv6, seed=1):
        super().__init__(series, points, block_rows, seed)
        from theia_b200 import anomaly_detection as ad
        from theia_b200 import clickhouse_native as chn
        self.enc = {}
        for name, ips in (("sourceIP", self.src_ip), ("destinationIP", self.dst_ip)):
            text = [ad.u32_to_ip(int(v)) for v in ips]
            if ipv6:
                text = ["fd00::%x:%x" % (int(v) >> 16, int(v) & 0xFFFF) if k % 5 == 0 else s
                        for k, (s, v) in enumerate(zip(text, ips))]
            enc = np.empty(len(text), dtype=object)
            enc[:] = [chn._enc_string(s) for s in text]
            self.enc[name] = enc

    def select_native_stream(self, sql):
        from theia_b200 import clickhouse_native as chn
        self.selects += 1
        spec = []
        for x in sql[len("SELECT "):sql.index(" FROM ")].split(", "):
            name = x.split(" AS ")[-1]
            spec.append((name, "UInt32" if x.startswith("IPv4StringToNum(") else TYPES.get(name, "String")))
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


class _Status:
    """The engine, keeping the status of every streamed job (main() only returns an exit code)."""

    def __init__(self, eng):
        self.eng, self.status = eng, []

    def __getattr__(self, name):
        return getattr(self.eng, name)

    def submit_stream(self, **kw):
        job = self.eng.submit_stream(**kw)
        wait = job.wait

        def keep(*a, **k):
            st = wait(*a, **k)
            self.status.append(st)
            return st
        job.wait = keep
        return job


def run_one(path, variant, series, points, block_rows):
    os.environ["TAD_STREAM_INPUT"] = "1"
    os.environ["TAD_IPV4_PUSHDOWN"] = "1" if path == "pushdown" else "0"
    os.environ["TAD_DEVICE_TEXT"] = "1" if path == "device-text" else "0"
    from theia_b200 import anomaly_detection as ad
    from theia_b200 import clickhouse_native as chn
    tr = TextTransport(series, points, block_rows, variant == "ipv6")
    out = {"variant": variant, "path": path, "block_rows": block_rows, "rows": tr.rows}
    rss0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    if path == "source":
        t0 = time.perf_counter()
        sql = ad.raw_select_sql(ad.plan_query())
        out["blocks"] = sum(1 for _ in chn.read_blocks_stream(tr.select_native_stream(sql)))
        wall = time.perf_counter() - t0
    else:
        from theia_b200.engine import TadEngine
        with TadEngine(device=0) as e:
            e.run({"flow_end": np.zeros(1, np.uint32), "value": np.ones(1, np.uint64)})     # context warm-up
            eng = _Status(e)
            rss0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
            t0 = time.perf_counter()
            assert ad.main(["--algo", "EWMA", "--id", "profile"], engine=eng, transport=tr) == 0
            wall = time.perf_counter() - t0
        st = eng.status[-1]
        out["h2d_ms"] = round(st["phase_ms"]["h2d"], 1)
        out["device_ms"] = round(st["device_ms"], 1)
        out["h2d_share"] = round(st["phase_ms"]["h2d"] / st["device_ms"], 3) if st["device_ms"] else None
        out["selects"] = tr.selects
        out["result_digest"] = _digest(tr.body)
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
    ap.add_argument("--variants", nargs="+", default=["ipv4", "ipv6"])
    ap.add_argument("--paths", nargs="+", default=["source", "host-dict", "device-text", "pushdown"])
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
                if path == "pushdown" and variant != "ipv4":
                    continue
                subprocess.run([sys.executable, os.path.abspath(__file__), "--run", "%s:%s" % (path, variant), "--series",
                                str(args.series), "--points", str(args.points), "--blocks", str(block)], check=True)


if __name__ == "__main__":
    main()
