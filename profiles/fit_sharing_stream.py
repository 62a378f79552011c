"""Fit sharing for streamed jobs (TAD_FLAG_SHARE, DESIGN.md section 8): the wall time of a job beside a long ARIMA fit
against the same job alone, and what the ARIMA job's detect phase, yields and parked time become, in both directions:
  * `stream_ewma`: a streamed EWMA job (--ewma-rows rows in 65,536-row host blocks, both addresses as text) submitted
    0.5 s into the fit phase of a tad_submit ARIMA job on a device-resident make_flows_torch(--series, 100, noisy=True)
    table;
  * `stream_arima`: a tad_submit EWMA job (2,000 x 100, device-resident) submitted 0.5 s into the fit phase of a streamed
    ARIMA job over the same long table in 65,536-row host blocks with text addresses, under a 1.5 GiB memory budget.
`alone_ms` is the job's submit-to-result time on an idle context (its feeder's time included for a streamed job);
`beside_ms` the same beside the fit, with sharing on (reserve 256 MiB) and the streamed job flagged.  The ARIMA job's
`detect_ms` (parked time left out), yields and parked time are given with sharing on and alone.
    python profiles/fit_sharing_stream.py [--series 150000] [--ewma-rows 2000000]
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
BLOCK = 65_536
RESERVE = 256 * MB
ARIMA_BUDGET = 1536 * MB


def _varuint(n):
    out = bytearray()
    while True:
        b = n & 0x7F
        n >>= 7
        out.append(b | (0x80 if n else 0))
        if not n:
            return bytes(out)


def text_blocks(table):
    """The table in host blocks with src_ip / dst_ip as Native String text ("fd00::<hex>") and its marks."""
    enc = {}
    for s in ("src_ip", "dst_ip"):
        uniq, inv = np.unique(table[s], return_inverse=True)
        e = np.array([_varuint(len(b"fd00::%x" % int(v))) + b"fd00::%x" % int(v) for v in uniq], dtype=object)
        enc[s] = (e, np.array([len(x) for x in e], dtype=np.uint64), inv)
    n = len(table["flow_end"])
    out = []
    for lo in range(0, n, BLOCK):
        hi = min(n, lo + BLOCK)
        b = {k: v[lo:hi] for k, v in table.items()}
        txt = {}
        for s, (e, lens, inv) in enc.items():
            i = inv[lo:hi]
            starts = np.zeros(hi - lo, dtype=np.uint64)
            np.cumsum(lens[i][:-1], out=starts[1:])
            txt[s] = (b"".join(e[i].tolist()), starts[::32].copy())
            b[s] = None
        out.append((b, txt))
    return out


def host_table(series, points, seed):
    from theia_b200 import synth
    t = synth.make_flows_torch(series, points, seed=seed, device="cuda", noisy=True)
    return {k: t[k].cpu().numpy().view(dt) for k, dt in synth.COLUMN_DTYPES.items()}


def device_table(series, points, seed):
    import torch
    from theia_b200 import synth
    from theia_b200.engine import DeviceColumns
    t = synth.make_flows_torch(series, points, seed=seed, device="cuda", noisy=True)
    torch.cuda.synchronize()
    d = DeviceColumns(int(t["value"].numel()), {k: v.data_ptr() for k, v in t.items()})
    d.keepalive = t
    return d


def feed(job, blocks):
    again = True
    while again:
        for b, txt in blocks:
            job.push(b, text=txt)
        again = job.end()


def start_stream(eng, blocks, **kw):
    job = eng.submit_stream(tad_id="stream", **kw)
    th = threading.Thread(target=feed, args=(job, blocks))
    th.start()
    return job, th


def wait_fitting(job):
    while job.progress()["fits_done"] == 0:
        time.sleep(0.001)


def timed(run):
    t0 = time.perf_counter()
    run()
    return (time.perf_counter() - t0) * 1e3


def arima_line(case, st, y, st_alone):
    return {"case": case, "job": "arima", "detect_ms": st["phase_ms"]["detect"],
            "detect_ms_alone": st_alone["phase_ms"]["detect"], "yields": y["yields"], "parked_ms": y["parked_ms"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=150_000)
    ap.add_argument("--ewma-rows", type=int, default=2_000_000)
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": smi}), flush=True)
    from theia_b200 import synth
    from theia_b200.engine import TadEngine
    long_dev = device_table(args.series, 100, 6)
    long_blocks = text_blocks(host_table(args.series, 100, 6))
    ewma_blocks = text_blocks(synth.make_flows(args.ewma_rows // 100, 100, seed=41))
    small_dev = device_table(2_000, 100, 13)
    with TadEngine(device=0) as eng:
        # ---- a streamed EWMA job beside a tad_submit ARIMA fit
        def stream_ewma(share):
            job, th = start_stream(eng, ewma_blocks, algo="EWMA", share=share)
            job.wait()
            th.join()
            job.release()
        stream_ewma(False)                                   # warm-up
        alone = timed(lambda: stream_ewma(False))
        job = eng.submit(long_dev, algo="ARIMA", tad_id="alone")
        st_alone = job.wait()
        job.release()
        eng.set_fit_sharing(RESERVE)
        job = eng.submit(long_dev, algo="ARIMA", tad_id="beside")
        wait_fitting(job)
        time.sleep(0.5)
        beside = timed(lambda: stream_ewma(True))
        running = job.poll()["state"] == "RUNNING"
        st = job.wait()
        y = job.yields()
        job.release()
        eng.set_fit_sharing(0)
        print(json.dumps({"case": "stream_ewma", "job": "ewma", "rows": args.ewma_rows, "alone_ms": alone,
                          "beside_ms": beside, "during_fit": running}), flush=True)
        print(json.dumps(arima_line("stream_ewma", st, y, st_alone)), flush=True)

        # ---- a tad_submit EWMA job beside a streamed ARIMA fit
        def ewma_job():
            q = eng.submit(small_dev, algo="EWMA", tad_id="q")
            q.wait()
            q.release()
        ewma_job()
        alone = timed(ewma_job)
        eng.set_memory_budget(ARIMA_BUDGET)
        hint = args.series * 100
        job, th = start_stream(eng, long_blocks, algo="ARIMA", rows_hint=hint)
        st_alone = job.wait()
        th.join()
        job.release()
        eng.set_fit_sharing(RESERVE)
        job, th = start_stream(eng, long_blocks, algo="ARIMA", rows_hint=hint, share=True)
        wait_fitting(job)
        time.sleep(0.5)
        beside = timed(ewma_job)
        running = job.poll()["state"] == "RUNNING"
        st = job.wait()
        th.join()
        y = job.yields()
        job.release()
        eng.set_fit_sharing(0)
        eng.set_memory_budget(0)
        print(json.dumps({"case": "stream_arima", "job": "ewma", "rows": 200_000, "alone_ms": alone, "beside_ms": beside,
                          "during_fit": running}), flush=True)
        print(json.dumps(arima_line("stream_arima", st, y, st_alone)), flush=True)


if __name__ == "__main__":
    main()
