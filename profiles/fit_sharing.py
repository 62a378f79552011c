"""Fit sharing (tad_set_fit_sharing, DESIGN.md section 8): the wait of an EWMA job queued behind an ARIMA fit, the ARIMA
fit rate alone and with k interleaves, and the cost of one yield.

    python profiles/fit_sharing.py --parent DIR [--rounds 3] [--series 50000] [--k 1 4 16]

DIR holds another build of the package (theia_b200/ with its libtheia_tad.so), e.g. the parent commit's; it is not part
of the repository.  Each run is a process of its own.  `rounds` times, alternating the two builds, a run times one
ARIMA job on a device-resident make_flows_torch(series, 100, noisy=True) table with sharing off (after a warm-up job):
`fits_per_s` is its records (one prefix fit per point) over the detect phase (Box-Cox, fits, scoring).  Then, with this
tree's build only:
  * latency: an EWMA job (2,000 x 100) submitted 0.5 s into the fit phase, from submit until its wait() returns, with
    sharing off and on (reserve 256 MiB);
  * interleaves: the ARIMA job with sharing on and k EWMA jobs spread over its fit phase; its detect phase (parked time
    excluded), its yields and parked time, and `yield_cost_ms` = (detect phase - the sharing-off detect phase) / yields:
    what one yield costs the fit (the fits dropped in flight and fitted again, and the resume launch).
Prints one JSON line per measurement, the card and its power limit first; writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MB = 1 << 20


def _table(series, points, seed):
    import torch
    from theia_b200 import synth
    from theia_b200.engine import DeviceColumns
    t = synth.make_flows_torch(series, points, seed=seed, device="cuda", noisy=True)
    torch.cuda.synchronize()
    d = DeviceColumns(int(t["value"].numel()), {k: v.data_ptr() for k, v in t.items()})
    d.keepalive = t
    return d


def _wait_fitting(job):
    while job.progress()["fits_done"] == 0:
        time.sleep(0.001)


def child_rate(args):
    from theia_b200.engine import TadEngine
    with TadEngine(device=0) as eng:
        cols = _table(args.series, 100, 6)
        for _ in range(2):
            job = eng.submit(cols, algo="ARIMA", tad_id="rate")
            st = job.wait()
            job.release()
        print(json.dumps({"build": args.build, "sharing": "off", "series": args.series, "detect_ms": st["phase_ms"]["detect"],
                          "fits_per_s": cols.c.rows / (st["phase_ms"]["detect"] * 1e-3)}))


def child_share(args):
    from theia_b200.engine import TadEngine
    with TadEngine(device=0) as eng:
        cols = _table(args.series, 100, 6)
        ewma = _table(2_000, 100, 13)
        job = eng.submit(cols, algo="ARIMA", tad_id="warm")
        st0 = job.wait()
        job.release()
        base = st0["phase_ms"]["detect"]
        for reserve in (0, 256 * MB):
            eng.set_fit_sharing(reserve)
            job = eng.submit(cols, algo="ARIMA", tad_id="latency")
            _wait_fitting(job)
            time.sleep(0.5)
            t0 = time.perf_counter()
            q = eng.submit(ewma, algo="EWMA", tad_id="queued")
            q.wait()
            lat = time.perf_counter() - t0
            q.release()
            job.wait()
            job.release()
            print(json.dumps({"measure": "ewma_latency", "sharing": "on" if reserve else "off", "latency_ms": lat * 1e3}))
        eng.set_fit_sharing(256 * MB)
        for k in [0] + args.k:
            job = eng.submit(cols, algo="ARIMA", tad_id="interleaves")
            _wait_fitting(job)
            for _ in range(k):
                time.sleep(base * 1e-3 / (k + 2))
                q = eng.submit(ewma, algo="EWMA", tad_id="interleaved")
                q.wait()
                q.release()
            st = job.wait()
            y = job.yields()
            job.release()
            det = st["phase_ms"]["detect"]
            print(json.dumps({"measure": "interleaves", "k": k, "yields": y["yields"], "parked_ms": y["parked_ms"],
                              "detect_ms": det, "detect_ms_sharing_off": base,
                              "fits_per_s": cols.c.rows / (det * 1e-3),
                              "yield_cost_ms": (det - base) / y["yields"] if y["yields"] else None}))
        eng.set_fit_sharing(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", required=True)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--series", type=int, default=50_000)
    ap.add_argument("--k", type=int, nargs="*", default=[1, 4, 16])
    ap.add_argument("--child", choices=["rate", "share"])
    ap.add_argument("--build", default="new")
    args = ap.parse_args()
    if args.child:
        sys.path.insert(0, ROOT if args.build == "new" else os.path.abspath(args.parent))
        (child_rate if args.child == "rate" else child_share)(args)
        return
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": smi}), flush=True)
    me = [sys.executable, os.path.abspath(__file__), "--parent", args.parent, "--series", str(args.series), "--k"] + \
        [str(k) for k in args.k]
    for _ in range(args.rounds):
        for build in ("parent", "new"):
            res = subprocess.run(me + ["--child", "rate", "--build", build], capture_output=True, text=True)
            sys.stdout.write(res.stdout if res.returncode == 0 else res.stdout + res.stderr[-3000:])
            sys.stdout.flush()
    res = subprocess.run(me + ["--child", "share"], capture_output=True, text=True)
    sys.stdout.write(res.stdout if res.returncode == 0 else res.stdout + res.stderr[-3000:])


if __name__ == "__main__":
    main()
