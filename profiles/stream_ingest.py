"""Rate of streamed input (DESIGN.md section 10): the BASELINE configs[1] table (1e8 rows / 1e6 connections x 100 points,
EWMA) pushed as pinned host blocks of 65,536 rows (ClickHouse's default block size) and of 8M rows, next to the same
table through the one-shot end-to-end path (tad_submit of pinned host columns), in the same run and on one context.

    python profiles/stream_ingest.py [--budgets-gb 0 3]

The blocks are views into one pinned copy of the table, so the figures are the engine's rate for blocks that are
already decoded; a decoding caller needs only two blocks of pinned memory (block_pinned_bytes).  Per budget (0 = none)
and block size: records/s submit -> result on the host, rounds, passes, peak device workspace, and whether the result
rows equal the unbudgeted one-shot run's bit for bit.  Prints one JSON line each, the card and its power limit first;
writes nothing."""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from profiles.memory_budget import card  # noqa: E402

ROW_BYTES = 29          # src_ip dst_ip src_port dst_port proto flow_start flow_end value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--budgets-gb", type=float, nargs="+", default=[0, 3], help="1e9 bytes; 0 = no budget")
    ap.add_argument("--blocks", type=int, nargs="+", default=[65536, 8 << 20])
    ap.add_argument("--series", type=int, default=1_000_000)
    ap.add_argument("--points", type=int, default=100)
    ap.add_argument("--steps", type=int, default=3)
    args = ap.parse_args()

    import numpy as np
    import torch
    from oracle import tad_oracle
    from theia_b200 import _lib as L
    from theia_b200 import synth
    from theia_b200.engine import TadEngine

    print(json.dumps(card()), flush=True)
    cols_t = synth.make_flows_torch(args.series, args.points, seed=1, device=torch.device("cuda", 0))
    rows = int(cols_t["value"].numel())
    widths = {"src_ip": 4, "dst_ip": 4, "src_port": 2, "dst_port": 2, "proto": 1, "flow_start": 4, "flow_end": 4,
              "value": 8}
    with TadEngine(device=0) as eng:
        hcols = eng.alloc_columns(rows)
        for name, t in cols_t.items():
            hv = hcols.view(name)
            hv[:rows] = t.cpu().numpy().view(hv.dtype)
        hcols.c.rows = rows
        del cols_t
        torch.cuda.empty_cache()

        def views(block_rows):
            for lo in range(0, rows, block_rows):
                c = L.TadColumns()
                c.rows = c.capacity = min(block_rows, rows - lo)
                c.mem = L.TAD_MEM_HOST
                for name, w in widths.items():
                    setattr(c, name, getattr(hcols.c, name) + lo * w)
                yield c

        def one_shot():
            job = eng.submit(hcols, algo="EWMA", tad_id="e2e")
            job.wait()
            return job

        def streamed(block_rows):
            job = eng.submit_stream(algo="EWMA", rows_hint=rows, tad_id="stream")
            rounds, again = 0, True
            while again:
                for c in views(block_rows):
                    rc = eng.lib.tad_stream_push(job.h, C.byref(c))
                    if rc != 0:
                        raise RuntimeError("tad_stream_push: %d %s" % (rc, job.poll()["err_msg"]))
                again = job.end()
                rounds += 1
            job.wait()
            job.rounds = rounds
            return job

        def leg(run, steps):
            t0, res, mem, rounds = time.perf_counter(), None, None, 1
            for k in range(steps):
                job = run()
                if k == steps - 1:
                    res, mem, rounds = job.result(), job.memory(), getattr(job, "rounds", 1)
                job.release()
            return rows * steps / (time.perf_counter() - t0), res, mem, rounds

        eng.set_memory_budget(0)
        leg(one_shot, 1)
        _, ref, _, _ = leg(one_shot, 1)
        ref = tad_oracle.canonicalize(ref)
        for gb in args.budgets_gb:
            budget = int(gb * 1e9)
            eng.set_memory_budget(budget)
            legs = [("e2e", None, one_shot)] + [("stream", b, (lambda b=b: streamed(b))) for b in args.blocks]
            for name, b, run in legs:
                leg(run, 1)
                rate, res, mem, rounds = leg(run, args.steps)
                res = tad_oracle.canonicalize(res)
                same = len(res["flow_end"]) == len(ref["flow_end"]) and all(
                    np.array_equal(res[c], ref[c], equal_nan=True) for c in ref)
                print(json.dumps({"budget_bytes": budget, "path": name, "block_rows": b, "rows": rows,
                                  "records_per_s": rate, "rounds": rounds, "passes": mem["passes"],
                                  "peak_workspace_bytes": mem["peak_workspace_bytes"],
                                  "block_pinned_bytes": 2 * b * ROW_BYTES if b else rows * ROW_BYTES,
                                  "result_rows": int(len(res["flow_end"])), "rows_equal_one_shot": bool(same)}),
                      flush=True)
        hcols.free()


if __name__ == "__main__":
    main()
