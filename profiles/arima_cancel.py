"""ARIMA fit throughput before and after the cancellable fit kernel, and the latency of a cancel during the fit phase
(DESIGN.md section 8, "Cancel and progress").

    python profiles/arima_cancel.py --parent DIR [--rounds 3] [--long 150000] [--long-points 4000] [--cancels 5]

DIR holds another build of the package (theia_b200/ with its libtheia_tad.so), e.g. the parent commit's, to compare
against; it is not part of the repository.  Each run is a process of its own, the two builds alternating `rounds` times.
A run times ARIMA jobs (emit_all) on two device-resident make_flows_torch(noisy=True) tables: the bench's ARIMA side-run
table (20,000 connections x 100 points, seed 5, after one warm-up job) and a long one (`long` x 100, seed 6).  It prints
records/s over the library's device time (`fits_per_s`: one prefix fit per point, as bench.py reports it) and over the
detect phase alone (`fits_per_s_detect`: Box-Cox, fits and scoring, without the host gaps of the pipeline), and a digest
of the sorted result rows, which must be the same for both builds.  Then, with this tree's build, `cancels` jobs on the
long table are cancelled 0.5 s into their fit phase, and `cancels` jobs on 2,000 x 100 points plus one connection of
`long_points` points 1 s into theirs (the short series are done by then: only the long one is being fitted): the time
from tad_cancel until wait() returns.  Prints one JSON line per run, the card and its power limit first; writes nothing."""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEY = ("src_ip", "dst_ip", "src_port", "dst_port", "proto", "flow_start", "flow_end")


def _table(series, seed, long_points=0):
    """make_flows_torch(series, 100, noisy=True), with one connection of `long_points` points appended (0: none)."""
    import torch
    from theia_b200 import synth
    from theia_b200.engine import DeviceColumns
    t = synth.make_flows_torch(series, 100, seed=seed, device="cuda", noisy=True)
    if long_points:
        one = synth.make_flows_torch(1, long_points, seed=seed + 1, device="cuda", noisy=True)
        t = {k: torch.cat([t[k], one[k]]).contiguous() for k in t}
    torch.cuda.synchronize()
    d = DeviceColumns(int(t["value"].numel()), {k: v.data_ptr() for k, v in t.items()})
    d.keepalive = t
    return d


def _digest(rows):
    import numpy as np
    order = np.lexsort([rows[k] for k in reversed(KEY)])
    h = hashlib.sha256()
    for k in sorted(rows):
        h.update(np.ascontiguousarray(rows[k][order]).tobytes())
    return h.hexdigest()[:16]


def child_throughput(args):
    from theia_b200.engine import TadEngine
    out = {"build": args.build}
    with TadEngine(device=0) as eng:
        for name, series, seed, warm in (("side", 20_000, 5, 1), ("long", args.long, 6, 0)):
            cols = _table(series, seed)
            for i in range(warm + 1):
                job = eng.submit(cols, algo="ARIMA", tad_id="profile", emit_all=True)
                st = job.wait()
                rows = job.result()
                job.release()
            out[name] = {"records": cols.c.rows, "fits_per_s": cols.c.rows / (st["device_ms"] * 1e-3),
                         "fits_per_s_detect": cols.c.rows / (st["phase_ms"]["detect"] * 1e-3),
                         "device_ms": st["device_ms"], "detect_ms": st["phase_ms"]["detect"],
                         "result_rows": st["result_rows"], "digest": _digest(rows)}
            del cols
    print(json.dumps(out))


def child_cancel(args):
    from theia_b200.engine import TadEngine
    with TadEngine(device=0) as eng:
        for name, cols, delay in (("long table", _table(args.long, 6), 0.5),
                                  ("long series", _table(2_000, 7, args.long_points), 1.0)):
            lat = []
            for _ in range(args.cancels):
                job = eng.submit(cols, algo="ARIMA", tad_id="cancel")
                while job.progress()["fits_done"] == 0:
                    time.sleep(0.002)
                time.sleep(delay)
                p = job.progress()
                t0 = time.perf_counter()
                job.cancel()
                st = job.wait(check=False)
                lat.append(time.perf_counter() - t0)
                assert st["state"] == "FAILED", st
                job.release()
                print(json.dumps({"table": name, "cancel_s": lat[-1], "fits_done_at_cancel": p["fits_done"],
                                  "fits_total": p["fits_total"]}))
            print(json.dumps({"table": name, "cancels": len(lat), "median_s": statistics.median(lat), "max_s": max(lat)}))
            del cols


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", required=True)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--long", type=int, default=150_000)
    ap.add_argument("--long-points", type=int, default=4000)
    ap.add_argument("--cancels", type=int, default=5)
    ap.add_argument("--child", choices=["throughput", "cancel"])
    ap.add_argument("--build", default="new")
    args = ap.parse_args()
    if args.child:
        sys.path.insert(0, ROOT if args.build == "new" else os.path.abspath(args.parent))
        (child_throughput if args.child == "throughput" else child_cancel)(args)
        return
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": smi}), flush=True)
    me = [sys.executable, os.path.abspath(__file__), "--parent", args.parent, "--long", str(args.long),
          "--long-points", str(args.long_points), "--cancels", str(args.cancels)]
    for r in range(args.rounds):
        for build in ("parent", "new"):
            res = subprocess.run(me + ["--child", "throughput", "--build", build], capture_output=True, text=True)
            sys.stdout.write(res.stdout if res.returncode == 0 else res.stdout + res.stderr[-3000:])
            sys.stdout.flush()
    res = subprocess.run(me + ["--child", "cancel"], capture_output=True, text=True)
    sys.stdout.write(res.stdout if res.returncode == 0 else res.stdout + res.stderr[-3000:])


if __name__ == "__main__":
    main()
