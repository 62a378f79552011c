"""Multi-GPU jobs in hash-range passes (DESIGN.md section 9, "Several GPUs"), one process per GPU:

    python -m torch.distributed.run --nproc-per-node 2 profiles/multi_gpu_passes.py --budgets-gb 0 40 12 6
    python -m torch.distributed.run --nproc-per-node 8 profiles/multi_gpu_passes.py --configs4 --budgets-gb 40

Default: BASELINE configs[1] rows per rank (1e6 connections x 100 points per GPU, EWMA) at each budget (0 = none, the
unplanned path), on a context of its own: device ms/step with device-resident input, e2e ms/step (submit -> result on the
host) with pinned host input, the passes every rank ran in and each rank's peak workspace, and whether the union of the
ranks' result rows equals that of the first budget bit for bit (compared through a digest on every rank).  --configs4:
configs[4] at its named size, 1.25e9 device-resident rows per GPU (1.25e7 connections x 100 per GPU), device ms only.
Rank 0 prints one JSON line per budget, the card and its power limit first; writes nothing."""
import argparse
import hashlib
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def digest(res):
    """Order-independent digest of one rank's result rows (canonical order, every column)."""
    from oracle import tad_oracle
    res = tad_oracle.canonicalize(res)
    h = hashlib.sha256()
    for c in sorted(res):
        h.update(res[c].tobytes())
    return h.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--budgets-gb", type=float, nargs="+", default=[0, 40, 12, 6], help="1e9 bytes per rank; 0 = none")
    ap.add_argument("--series-per-gpu", type=int, default=1_000_000)
    ap.add_argument("--points", type=int, default=100)
    ap.add_argument("--configs4", action="store_true", help="1.25e7 connections x 100 points per GPU, device input only")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()

    import torch
    import torch.distributed as dist
    from profiles.memory_budget import card
    from theia_b200 import synth
    from theia_b200.engine import DeviceColumns, TadEngine

    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    dist.init_process_group("gloo")
    if not torch.cuda.is_available() or torch.cuda.device_count() <= local:
        raise SystemExit("rank %d: no GPU %d; this measurement needs one GPU per rank" % (rank, local))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    series = 12_500_000 if args.configs4 else args.series_per_gpu
    if rank == 0:
        print(json.dumps(dict(card(), world=world, series_per_gpu=series, points=args.points)), flush=True)
    cols_t = synth.make_flows_torch_sharded(series, args.points, seed=4, device=dev, rank=rank, world=world)
    rows = int(cols_t["value"].numel())
    total = sum(dist_all(dist, world, rows))
    torch.cuda.synchronize()
    dcols = DeviceColumns(rows, {k: v.data_ptr() for k, v in cols_t.items()})
    dcols.keepalive = cols_t
    first = None
    for gb in args.budgets_gb:
        budget = int(gb * 1e9)
        uid = [TadEngine.get_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, src=0)
        with TadEngine(device=local, world_size=world, rank=rank, nccl_unique_id=uid[0], memory_budget=budget) as eng:
            def leg(cols, steps):
                dev_ms, mem, res = 0.0, None, None
                dist.barrier()
                t0 = time.perf_counter()
                for k in range(steps):
                    job = eng.submit(cols, algo="EWMA", tad_id="mgpasses", global_rows=total)
                    st = job.wait()
                    dev_ms += st["device_ms"]
                    mem = job.memory()
                    res = job.result() if k == steps - 1 else None
                    job.release()
                return dev_ms / steps, (time.perf_counter() - t0) * 1e3 / steps, mem, res

            leg(dcols, args.warmup)
            ms_dev, _, mem, res = leg(dcols, args.steps)
            ms_e2e = None
            if not args.configs4:
                hcols = eng.alloc_columns(rows)
                for name, t in cols_t.items():
                    hv = hcols.view(name)
                    hv[:rows] = t.cpu().numpy().view(hv.dtype)
                hcols.c.rows = rows
                leg(hcols, args.warmup)
                _, ms_e2e, _, _ = leg(hcols, args.steps)
                hcols.free()
        d = digest(res)
        if first is None:
            first = d
        line = dist_all(dist, world, dict(passes=mem["passes"], peak=mem["peak_workspace_bytes"], dev=ms_dev, e2e=ms_e2e,
                                           same=d == first))
        if rank == 0:
            print(json.dumps({"budget_bytes_per_rank": budget, "rows_per_rank": rows,
                              "passes": [x["passes"] for x in line],
                              "peak_workspace_bytes": [x["peak"] for x in line],
                              "device_ms_per_step": max(x["dev"] for x in line),
                              "e2e_ms_per_step": None if ms_e2e is None else max(x["e2e"] for x in line),
                              "rows_equal_first_budget": all(x["same"] for x in line)}), flush=True)
    dist.barrier()
    dist.destroy_process_group()


def dist_all(dist, world, x):
    got = [None] * world
    dist.all_gather_object(got, x)
    return got


if __name__ == "__main__":
    main()
