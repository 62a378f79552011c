"""Time of each capacity class of the group kernel at the bench shape (DESIGN.md section 4):

    python profiles/group_classes.py [--steps 5] [--warmup 3]

Runs the bench job -- 1e6 connections x 100 points, device-resident input, EWMA -- warm-up steps first, then the timed
steps under torch.profiler (CUDA activities; a run of its own, so profile overheads stay out of bench.py's numbers).
Every `group_kernel<CAP, NT, MODE>` instance shows up under its own name.  For each one the script prints, per step, its
kernel time and share of the group phase, and the buckets and rows of its class: the buckets holding more rows than the
next smaller class and at most CAP, counted from the host mirror of the engine's key hash and bucket count
(theia_b200/sharding.py).
Prints one JSON line, the card and its power limit first; writes nothing."""
import argparse
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series", type=int, default=1_000_000)
    ap.add_argument("--points", type=int, default=100)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    from profiles.memory_budget import card
    from theia_b200 import sharding, synth
    from theia_b200.engine import DeviceColumns, TadEngine

    if not torch.cuda.is_available():
        raise SystemExit("no GPU: this measurement needs one")
    dev = torch.device("cuda", 0)
    cols_t = synth.make_flows_torch(args.series, args.points, seed=1, device=dev)      # bench.py's table
    rows = int(cols_t["value"].numel())
    logb = sharding.pick_logb(rows)
    bucket = sharding.key_hash(synth.torch_cols_to_numpy(cols_t)) >> np.uint64(64 - logb)
    hist = np.bincount(bucket.astype(np.int64), minlength=1 << logb)
    dcols = DeviceColumns(rows, {k: v.data_ptr() for k, v in cols_t.items()})
    dcols.keepalive = cols_t

    with TadEngine(device=0) as eng:
        def step():
            job = eng.submit(dcols, algo="EWMA", tad_id="groupclasses")
            st = job.wait()
            job.release()
            return st

        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                step()
            torch.cuda.synchronize()

    per = {}
    for ev in prof.key_averages():
        m = re.search(r"group_kernel<(\d+), (\d+), (\d+)>", ev.key)
        if m:
            cap, nt, mode = (int(g) for g in m.groups())
            k = (cap, nt, mode)
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            per[k] = per.get(k, 0.0) + t / 1e3 / args.steps
    caps = sorted({k[0] for k in per})
    total = sum(per.values())
    out = []
    for k in sorted(per):
        cap = k[0]
        lo = max([c for c in caps if c < cap], default=0)
        sel = (hist > lo) & (hist <= cap)
        out.append({"kernel": "group_kernel<%d, %d, %d>" % k, "rows_lo": lo, "rows_hi": cap,
                    "ms_per_step": per[k], "share": per[k] / total if total else None,
                    "buckets": int(sel.sum()), "rows": int(hist[sel].sum())})
    print(json.dumps(dict(card(), rows=rows, buckets=1 << logb, steps=args.steps, group_ms_per_step=total,
                          spilled_buckets=int((hist > max(caps, default=0)).sum()), classes=out)), flush=True)


if __name__ == "__main__":
    main()
