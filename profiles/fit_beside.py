"""Fitting beside a fit (TAD_FLAG_FIT_BESIDE, DESIGN.md section 8): the wait of an ARIMA job B queued behind an ARIMA fit
A, with and without the flag, and what B's fit beside it costs A; the sharing-off fit rate and the bench line of this
build against another.

    python profiles/fit_beside.py --parent DIR [--rounds 3] [--series 50000] [--b-series 2000] [--what rate bench beside]

DIR holds another build of the package (theia_b200/ with its libtheia_tad.so, and its bench.py), e.g. the parent
commit's; it is not part of the repository.  Each run is a process of its own.  `rounds` times, alternating the two
builds (`--what` picks the parts, all by default):
  * rate: one ARIMA job on a device-resident make_flows_torch(series, 100, noisy=True) table with sharing off (after a
    warm-up job): `fits_per_s` is its records (one prefix fit per point) over the detect phase;
  * bench: `bench.py --gpus 1 --steps 5 --warmup 2 --no-parity` of that build, its JSON line.
Then, with this tree's build only, B (b_series x 100) is timed alone, and then submitted 0.5 s into A's fit phase
(sharing on, reserve 256 MiB), without and with the flag: B's submit-to-complete time, and A's detect phase (parked time
left out), yields and parked time.
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


def child_beside(args):
    from theia_b200.engine import TadEngine
    with TadEngine(device=0) as eng:
        a_cols = _table(args.series, 100, 6)
        b_cols = _table(args.b_series, 100, 21)
        for _ in range(2):
            t0 = time.perf_counter()
            q = eng.submit(b_cols, algo="ARIMA", tad_id="B-solo")
            st_b = q.wait()
            solo = time.perf_counter() - t0
            q.release()
        job = eng.submit(a_cols, algo="ARIMA", tad_id="A-solo")
        st_a = job.wait()
        job.release()
        print(json.dumps({"measure": "solo", "b_series": args.b_series, "b_ms": solo * 1e3,
                          "b_detect_ms": st_b["phase_ms"]["detect"], "a_series": args.series,
                          "a_detect_ms": st_a["phase_ms"]["detect"]}))
        eng.set_fit_sharing(256 * MB)
        for beside in (False, True):
            job = eng.submit(a_cols, algo="ARIMA", tad_id="A")
            _wait_fitting(job)
            time.sleep(0.5)
            t0 = time.perf_counter()
            q = eng.submit(b_cols, algo="ARIMA", tad_id="B", fit_beside=beside)
            q.wait()
            wait = time.perf_counter() - t0
            yb = q.yields()
            q.release()
            st = job.wait()
            y = job.yields()
            job.release()
            print(json.dumps({"measure": "b_behind_a", "fit_beside": beside, "b_ms": wait * 1e3,
                              "b_yields": yb["yields"], "a_detect_ms": st["phase_ms"]["detect"],
                              "a_detect_ms_solo": st_a["phase_ms"]["detect"], "a_yields": y["yields"],
                              "a_parked_ms": y["parked_ms"]}))
        eng.set_fit_sharing(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", required=True)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--series", type=int, default=50_000)
    ap.add_argument("--b-series", type=int, default=2_000)
    ap.add_argument("--what", nargs="*", choices=["rate", "bench", "beside"], default=["rate", "bench", "beside"])
    ap.add_argument("--child", choices=["rate", "beside"])
    ap.add_argument("--build", default="new")
    args = ap.parse_args()
    if args.child:
        sys.path.insert(0, ROOT if args.build == "new" else os.path.abspath(args.parent))
        (child_rate if args.child == "rate" else child_beside)(args)
        return
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": smi}), flush=True)
    me = [sys.executable, os.path.abspath(__file__), "--parent", args.parent, "--series", str(args.series),
          "--b-series", str(args.b_series)]

    def run(cmd, tag=None):
        res = subprocess.run(cmd, capture_output=True, text=True)
        out = res.stdout if res.returncode == 0 else res.stdout + res.stderr[-3000:]
        if tag:
            out = "".join(json.dumps({"build": tag, "bench": json.loads(l)}) + "\n" if l.startswith("{") else l + "\n"
                          for l in out.splitlines())
        sys.stdout.write(out)
        sys.stdout.flush()

    for _ in range(args.rounds):
        for build in ("parent", "new"):
            if "rate" in args.what:
                run(me + ["--child", "rate", "--build", build])
            if "bench" in args.what:
                tree = ROOT if build == "new" else os.path.abspath(args.parent)
                run([sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", "5", "--warmup", "2",
                     "--no-parity"], build)
    if "beside" in args.what:
        run(me + ["--child", "beside"])


if __name__ == "__main__":
    main()
