"""A streamed ARIMA job fitting beside a fit (TAD_FLAG_SHARE | TAD_FLAG_FIT_BESIDE, DESIGN.md section 8): the wait of a
streamed ARIMA job B queued behind an ARIMA fit A, with both flags and with TAD_FLAG_SHARE only, and what B's fit beside
it costs A.
  * A: an ARIMA job on make_flows_torch(--series, 100, noisy=True), once tad_submit on the device-resident table and
    once streamed, the same table in 65,536-row host blocks with both addresses as text;
  * B: a streamed ARIMA job on make_flows_torch(--b-series, 100, noisy=True) in 65,536-row host blocks with text
    addresses, its feeder started 0.5 s into A's fit phase, sharing on with a 256 MiB reserve.
`b_ms` is B's submit-to-result time (its feeder's time included); `b_alone_ms` the same on an idle context.  A's
`detect_ms` (parked time left out; its fit phase) is given beside B and alone, with its yields and parked time.
    python profiles/fit_beside_stream.py [--series 50000] [--b-series 2000]
Prints one JSON line per measurement, the card and its power limit first; writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from fit_sharing_stream import device_table, host_table, start_stream, text_blocks, timed, wait_fitting  # noqa: E402

MB = 1 << 20
RESERVE = 256 * MB


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=50_000)
    ap.add_argument("--b-series", type=int, default=2_000)
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": smi}), flush=True)
    from theia_b200.engine import TadEngine
    a_dev = device_table(args.series, 100, 6)
    a_blocks = text_blocks(host_table(args.series, 100, 6))
    b_blocks = text_blocks(host_table(args.b_series, 100, 21))
    hint = args.series * 100
    with TadEngine(device=0) as eng:
        def start_a(streamed, tad_id, share=False):
            if streamed:
                return start_stream(eng, a_blocks, algo="ARIMA", rows_hint=hint, share=share)
            return eng.submit(a_dev, algo="ARIMA", tad_id=tad_id), None

        def run_b(**flags):
            job, th = start_stream(eng, b_blocks, algo="ARIMA", **flags)
            job.wait()
            th.join()
            y = job.yields()
            job.release()
            return y

        run_b()                                              # warm-up
        b_alone = timed(run_b)
        for streamed in (False, True):
            mode = "stream" if streamed else "submit"
            job, th = start_a(streamed, "A-alone")
            st_alone = job.wait()
            if th:
                th.join()
            job.release()
            for beside in (True, False):
                eng.set_fit_sharing(RESERVE)
                job, th = start_a(streamed, "A", share=True)
                wait_fitting(job)
                time.sleep(0.5)
                yb = {}
                b_ms = timed(lambda: yb.update(run_b(share=True, fit_beside=beside)))
                running = job.poll()["state"] == "RUNNING"
                st = job.wait()
                if th:
                    th.join()
                y = job.yields()
                job.release()
                eng.set_fit_sharing(0)
                print(json.dumps({"a": mode, "a_series": args.series, "b_series": args.b_series,
                                  "b_flags": "share|fit_beside" if beside else "share", "b_ms": b_ms,
                                  "b_alone_ms": b_alone, "b_yields": yb["yields"], "a_running_at_b_end": running,
                                  "a_detect_ms": st["phase_ms"]["detect"],
                                  "a_detect_ms_alone": st_alone["phase_ms"]["detect"],
                                  "a_yields": y["yields"], "a_parked_ms": y["parked_ms"]}), flush=True)


if __name__ == "__main__":
    main()
