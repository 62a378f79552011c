"""Jobs streamed to every rank (TAD_FLAG_RANK_STREAM, DESIGN.md section 10, "Several GPUs"), one process per GPU:

    python -m torch.distributed.run --nproc-per-node 2 profiles/multi_gpu_stream.py
    python -m torch.distributed.run --nproc-per-node 8 profiles/multi_gpu_stream.py --configs4 --budget-gb 40

Default: configs[1]-shape shards per rank (1e6 connections x 100 points per GPU, EWMA), streamed from pinned host blocks
of 65,536 rows and of 8M rows, next to the one-shot rank job (tad_submit of the same shard from pinned host columns).
--configs4: configs[4] at its named size, 1.25e9 rows per GPU streamed from device blocks of 8M rows generated block by
block, so no rank holds its shard anywhere.  Per leg: device ms, wall ms, rounds, passes (every rank), and the peak host
RSS of every rank.  Rank 0 prints one JSON line per leg, the card and its power limit first; writes nothing."""
import argparse
import json
import os
import resource
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--series-per-gpu", type=int, default=1_000_000)
    ap.add_argument("--points", type=int, default=100)
    ap.add_argument("--configs4", action="store_true", help="1.25e7 connections x 100 points per GPU from device blocks")
    ap.add_argument("--budget-gb", type=float, default=0, help="1e9 bytes per rank; 0 = free memory less the headroom")
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
    uid = [TadEngine.get_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    eng = TadEngine(device=local, world_size=world, rank=rank, nccl_unique_id=uid[0], memory_budget=int(args.budget_gb * 1e9))

    def gather(x):
        got = [None] * world
        dist.all_gather_object(got, x)
        return got

    def report(name, st, wall_ms, rounds, passes):
        line = gather(dict(dev=st["device_ms"], wall=wall_ms, rounds=rounds, passes=passes,
                           rss=resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024))
        if rank == 0:
            print(json.dumps({"leg": name, "rows_per_rank": rows, "device_ms": max(x["dev"] for x in line),
                              "wall_ms": max(x["wall"] for x in line), "rounds": [x["rounds"] for x in line],
                              "passes": [x["passes"] for x in line], "peak_rss_bytes": [x["rss"] for x in line]}),
                  flush=True)

    def stream(name, blocks, hint):
        """blocks(): one round's blocks; every rank feeds its own job from this thread."""
        dist.barrier()
        t0 = time.perf_counter()
        job = eng.submit_stream(algo="EWMA", tad_id="mgstream", rows_hint=hint, ranks=True)
        rounds = 0
        while True:
            for b in blocks():
                job.push(b)
            rounds += 1
            if not job.end():
                break
        st = job.wait()
        passes = job.memory()["passes"]
        job.release()
        report(name, st, (time.perf_counter() - t0) * 1e3, rounds, passes)

    if args.configs4:
        rows = series * args.points
        per_block = 8 << 20
        n_blocks = (rows + per_block - 1) // per_block

        def gen_blocks():
            # block k: connections [k * per_block / points, ...) of this rank, generated on the device as it is needed
            s_per = per_block // args.points
            for k in range(n_blocks):
                n = min(s_per, series - k * s_per)
                if n <= 0:
                    return
                t = synth.make_flows_torch_sharded(n, args.points, seed=4 + k, device=dev, rank=rank, world=world)
                torch.cuda.synchronize()
                d = DeviceColumns(int(t["value"].numel()), {c: v.data_ptr() for c, v in t.items()})
                d.keepalive = t
                yield d
        stream("configs4_device_8M", gen_blocks, rows)
    else:
        cols_t = synth.make_flows_torch_sharded(series, args.points, seed=4, device=dev, rank=rank, world=world)
        rows = int(cols_t["value"].numel())
        hcols = eng.alloc_columns(rows)
        for name, t in cols_t.items():
            hv = hcols.view(name)
            hv[:rows] = t.cpu().numpy().view(hv.dtype)
        hcols.c.rows = rows
        del cols_t
        torch.cuda.empty_cache()
        dist.barrier()
        t0 = time.perf_counter()
        job = eng.submit(hcols, algo="EWMA", tad_id="mgstream-ref")
        st = job.wait()
        passes = job.memory()["passes"]
        job.release()
        report("one_shot_host", st, (time.perf_counter() - t0) * 1e3, 0, passes)
        for per_block in (65_536, 8 << 20):
            bufs = [eng.alloc_columns(per_block) for _ in range(2)]

            def host_blocks():
                for k, lo in enumerate(range(0, rows, per_block)):
                    hi = min(rows, lo + per_block)
                    b = bufs[k & 1]           # free again: the push of block k - 1 has returned
                    for name in ("src_ip", "dst_ip", "src_port", "dst_port", "proto", "flow_start", "flow_end", "value"):
                        b.view(name)[:hi - lo] = hcols.view(name)[lo:hi]
                    b.c.rows = hi - lo
                    yield b
            stream("host_%d" % per_block, host_blocks, rows)
            for b in bufs:
                b.free()
        hcols.free()
    eng.close()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
