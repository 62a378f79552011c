"""Lending (TAD_FLAG_LEND, DESIGN.md section 10): queued EWMA jobs beside a streamed job whose caller is slower than the GPU.
A configs[1]-shaped streamed EWMA job (--rows rows, 100 points per connection) is fed from two pinned host blocks of
--block rows at a throttled source rate (--rate rows/s, near the job entry's measured rates), while a 1e6-row EWMA
tad_submit job (pinned host columns) is submitted every --every ms.  Fit sharing is on (reserve 256 MiB) in both arms;
the only difference is the streamed job's TAD_FLAG_LEND.  Per arm: the queued jobs' submit-to-complete latency (median,
maximum), the streamed job's wall time from submit to result and its lent() counts.  `alone_ms` is one queued job on an
idle context.
    python profiles/stream_lend.py [--rows 10000000] [--rate 5e6] [--block 65536] [--every 200] [--reps 2]
Prints one JSON line per measurement, the card and its power limit first; writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
MB = 1 << 20
RESERVE = 256 * MB


def host_table(series, points, seed):
    from theia_b200 import synth
    t = synth.make_flows_torch(series, points, seed=seed, device="cuda", noisy=True)
    return {k: t[k].cpu().numpy().view(dt) for k, dt in synth.COLUMN_DTYPES.items()}


def run_arm(eng, table, queued_cols, args, lend):
    """One streamed job fed at the source rate, queued jobs submitted meanwhile: the arm's JSON record."""
    n = len(table["flow_end"])
    ring = [eng.alloc_columns(args.block), eng.alloc_columns(args.block)]
    jobs, stop = [], threading.Event()

    def submitter():
        while not stop.is_set():
            jobs.append(eng.submit(queued_cols, algo="EWMA", tad_id="queued"))
            stop.wait(args.every / 1e3)

    t0 = time.perf_counter()
    job = eng.submit_stream(algo="EWMA", tad_id="stream", rows_hint=n, lend=lend)
    th = threading.Thread(target=submitter)
    th.start()
    try:
        k = 0
        for lo in range(0, n, args.block):
            hi = min(n, lo + args.block)
            due = t0 + hi / args.rate                      # the source delivers rows [lo, hi) by then
            c = ring[k % 2].fill({name: v[lo:hi] for name, v in table.items()})
            wait = due - time.perf_counter()
            if wait > 0:
                time.sleep(wait)
            job.push(c)
            k += 1
        assert not job.end()
        job.wait()
        wall_ms = (time.perf_counter() - t0) * 1e3
        stop.set()
        th.join()
        lent = job.lent()
        lat = []
        for q in jobs:
            lat.append(q.wait()["total_ms"])
            q.release()
    finally:
        stop.set()
        th.join()
        job.release()
        for c in ring:
            c.free()
    lat = np.array(lat)
    return {"lend": lend, "stream_wall_ms": round(wall_ms, 1), "source_ms": round(n / args.rate * 1e3, 1),
            "queued_jobs": len(lat), "queued_median_ms": round(float(np.median(lat)), 2),
            "queued_max_ms": round(float(lat.max()), 2), "lent_jobs": lent["jobs_run"],
            "lent_ms": round(lent["lent_ms"], 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--rate", type=float, default=5e6)
    ap.add_argument("--block", type=int, default=65_536)
    ap.add_argument("--every", type=float, default=200.0)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": smi}), flush=True)
    from theia_b200 import synth
    from theia_b200.engine import TadEngine
    table = host_table(args.rows // 100, 100, 7)
    with TadEngine(device=0) as eng:
        queued_cols = eng.columns_from_numpy(synth.make_flows(10_000, 100, seed=8))
        alone = []
        for _ in range(5):
            q = eng.submit(queued_cols, algo="EWMA", tad_id="alone")
            alone.append(q.wait()["total_ms"])
            q.release()
        print(json.dumps({"alone_ms": round(float(np.median(alone[1:])), 2)}), flush=True)
        eng.set_fit_sharing(RESERVE)
        run_arm(eng, table, queued_cols, args, False)       # warm-up: pinned pools, first-touch of the workspace
        for _ in range(args.reps):
            for lend in (False, True):
                rec = run_arm(eng, table, queued_cols, args, lend)
                rec.update(rows=args.rows, rate=args.rate, block=args.block, every_ms=args.every)
                print(json.dumps(rec), flush=True)
        eng.set_fit_sharing(0)
        queued_cols.free()


if __name__ == "__main__":
    main()
