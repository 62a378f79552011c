"""Cost of the memory budget (DESIGN.md section 9): the BASELINE configs[1] table (1e8 rows / 1e6 connections x 100 points,
EWMA) at several device memory budgets, each on a context of its own.

    python profiles/memory_budget.py --budgets-gb 0 40 6 3 1.5

Per budget (0 = none): device ms/step with device-resident input, e2e ms/step (submit -> result on the host) with pinned
host input, the passes each ran in, the peak workspace, and whether the result rows equal those of the run without a
budget bit for bit.  Prints one JSON line per budget, the card and its power limit first; writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:          # the numbers are still printed; the card is then unknown
        return {"gpu": None, "error": repr(e)[:200]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--budgets-gb", type=float, nargs="+", default=[0, 40, 6, 3, 1.5], help="1e9 bytes; 0 = no budget")
    ap.add_argument("--series", type=int, default=1_000_000)
    ap.add_argument("--points", type=int, default=100)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    import numpy as np
    import torch
    from oracle import tad_oracle
    from theia_b200 import synth
    from theia_b200.engine import DeviceColumns, TadEngine

    print(json.dumps(card()), flush=True)
    dev = torch.device("cuda", 0)
    cols_t = synth.make_flows_torch(args.series, args.points, seed=1, device=dev)
    rows = int(cols_t["value"].numel())
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    dcols = DeviceColumns(rows, {k: v.data_ptr() for k, v in cols_t.items()})
    dcols.keepalive = cols_t
    ref = None
    for gb in args.budgets_gb:
        budget = int(gb * 1e9)
        with TadEngine(device=0, memory_budget=budget) as eng:
            hcols = eng.alloc_columns(rows)
            for name, t in cols_t.items():
                hv = hcols.view(name)
                hv[:rows] = t.cpu().numpy().view(hv.dtype)
            hcols.c.rows = rows

            def leg(cols, steps):
                dev_ms, t0, mem, res = 0.0, time.perf_counter(), None, None
                for k in range(steps):
                    job = eng.submit(cols, algo="EWMA", tad_id="budget")
                    st = job.wait()
                    dev_ms += st["device_ms"]
                    mem = job.memory()
                    if k == steps - 1:
                        res = job.result()
                    else:
                        job.result(copy=False)
                    job.release()
                return dev_ms / steps, (time.perf_counter() - t0) * 1e3 / steps, mem, res

            leg(dcols, args.warmup)
            ms_dev, _, mem_dev, res = leg(dcols, args.steps)
            leg(hcols, max(1, args.warmup // 2))
            _, ms_e2e, mem_e2e, _ = leg(hcols, args.steps)
            hcols.free()
        res = tad_oracle.canonicalize(res)
        if ref is None:
            ref = res
        same = len(res["flow_end"]) == len(ref["flow_end"]) and all(
            np.array_equal(res[c], ref[c], equal_nan=True) for c in ref)
        print(json.dumps({"budget_bytes": budget, "rows": rows, "device_ms_per_step": ms_dev, "e2e_ms_per_step": ms_e2e,
                          "passes": mem_dev["passes"], "peak_workspace_bytes": mem_dev["peak_workspace_bytes"],
                          "e2e_passes": mem_e2e["passes"], "e2e_peak_workspace_bytes": mem_e2e["peak_workspace_bytes"],
                          "result_rows": int(len(res["flow_end"])), "rows_equal_first_budget": bool(same)}), flush=True)


if __name__ == "__main__":
    main()
