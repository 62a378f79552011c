"""Host row store (DESIGN.md section 11): the BASELINE configs[1] table (1e8 rows / 1e6 connections x 100 points, EWMA)
streamed as pinned host blocks of 65,536 rows (ClickHouse's default block size) and of 8M rows, under device budgets of
3 GB and 1.5 GB, each without a host row store and with one large enough for the round.

    python profiles/host_store.py [--budgets-gb 3 1.5] [--host-gb 0 3.6]

The blocks are views into one pinned copy of the table, as in profiles/stream_ingest.py: already decoded, so the figures
leave out what a round costs a real source (a ClickHouse scan and the decode of its String columns), which is what the
store saves.  Per run: records/s submit -> result on the host, rounds and the rows the caller delivered, passes, peak
device workspace and peak store bytes, and whether the result rows equal the unbudgeted one-shot run's bit for bit.
Prints one JSON line each, the card and its power limit first; writes nothing."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--budgets-gb", type=float, nargs="+", default=[3, 1.5], help="device budgets, 1e9 bytes")
    ap.add_argument("--host-gb", type=float, nargs="+", default=[0, 3.6], help="host budgets, 1e9 bytes; 0 = no store")
    ap.add_argument("--blocks", type=int, nargs="+", default=[65536, 8 << 20])
    ap.add_argument("--series", type=int, default=1_000_000)
    ap.add_argument("--points", type=int, default=100)
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

        def canon(job):
            return tad_oracle.canonicalize(job.result())

        eng.set_memory_budget(0)
        job = eng.submit(hcols, algo="EWMA", tad_id="one-shot")
        job.wait()
        ref = canon(job)
        job.release()

        def streamed(block_rows):
            t0 = time.perf_counter()
            job = eng.submit_stream(algo="EWMA", rows_hint=rows, tad_id="stream")
            rounds, delivered, again = 0, 0, True
            while again:
                for c in views(block_rows):
                    rc = eng.lib.tad_stream_push(job.h, C.byref(c))
                    if rc != 0:
                        raise RuntimeError("tad_stream_push: %d %s" % (rc, job.poll()["err_msg"]))
                    delivered += c.rows
                again = job.end()
                rounds += 1
            st = job.wait()
            dt = time.perf_counter() - t0
            return job, st, rounds, delivered, dt

        # host budget outermost: the context keeps its store pages from job to job, so the first job with a store pins
        # them ("warm": false) and the later ones reuse them
        for hgb in args.host_gb:
            eng.set_host_budget(int(hgb * 1e9))
            warm = False
            for gb in args.budgets_gb:
                eng.set_memory_budget(int(gb * 1e9))
                for b in args.blocks:
                    job, st, rounds, delivered, dt = streamed(b)
                    mem = job.memory()
                    res = canon(job)
                    job.release()
                    same = len(res["flow_end"]) == len(ref["flow_end"]) and all(
                        np.array_equal(res[c], ref[c], equal_nan=True) for c in ref)
                    print(json.dumps({"budget_bytes": int(gb * 1e9), "host_budget_bytes": int(hgb * 1e9), "warm": warm,
                                      "block_rows": b, "rows": rows, "records_per_s": rows / dt, "rounds": rounds,
                                      "rows_delivered": delivered, "passes": mem["passes"],
                                      "stored_rows": mem["stored_rows"],
                                      "peak_workspace_bytes": mem["peak_workspace_bytes"],
                                      "peak_host_bytes": mem["peak_host_bytes"], "h2d_ms": st["phase_ms"]["h2d"],
                                      "device_ms": st["device_ms"], "rows_equal_one_shot": bool(same)}), flush=True)
                    warm = hgb > 0
        eng.set_host_budget(0)
        hcols.free()


if __name__ == "__main__":
    main()
