"""Worker of tests/test_gpu_multi_rank_passes.py: multi-GPU jobs in hash-range passes under a memory budget (launched with
torch.distributed.run, one process per rank).

    python -m torch.distributed.run --nproc-per-node N tests/multi_passes_worker.py <out_dir>

Every rank runs its row shard of every case and saves its result rows (res_<case>_<rank>.npz) and its status
(st_<case>_<rank>.json); the parent test compares the union over the ranks with the oracle and with the no-budget run.
Checks that need every rank's view (the same pass count everywhere, the same verdict everywhere) are made here."""
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from theia_b200 import sharding, synth  # noqa: E402

MB = 1 << 20
BUDGET_2 = 200 * MB          # 2M rows per rank: two passes or more
BUDGET_4 = 64 * MB           # the floor: four passes or more
ROOMY = 1024 * MB
_SIGNED = {np.dtype(np.uint32): np.int32, np.dtype(np.uint16): np.int16, np.dtype(np.uint64): np.int64,
           np.dtype(np.uint8): np.uint8}


def case_table(name, world):
    """The same table on every rank."""
    if name == "spread":                                       # 2M rows per rank, every owner about as large
        return synth.make_flows(20000 * world, 100, seed=81)
    if name == "skewed":                                       # the last rank owns about three times its share
        base = synth.make_flows(10000 * world, 100, seed=82)
        extra = synth.make_flows(20000 * world, 100, seed=83)
        keep = sharding.owner_rank(extra, world, len(extra["value"]) + len(base["value"])) == world - 1
        t = {k: np.concatenate([base[k], extra[k][keep]]) for k in base}
        perm = np.random.default_rng(84).permutation(len(t["value"]))
        return {k: v[perm] for k, v in t.items()}
    if name == "one_big":                                      # one connection of 2M points: no 1/64 range fits 64 MiB
        small = synth.make_flows(2000, 50, seed=85)
        big = synth.make_flows(1, 2_000_000, seed=86)
        return {k: np.concatenate([small[k], big[k]]) for k in small}
    if name == "small":
        return synth.make_flows(3000 * world, 30, seed=87)
    raise KeyError(name)


def device_cols(table):
    from theia_b200.engine import DeviceColumns
    ts = {k: torch.from_numpy(np.ascontiguousarray(v).view(_SIGNED[v.dtype])).cuda() for k, v in table.items()
          if v is not None and k not in ("src_ns", "dst_ns")}
    d = DeviceColumns(len(table["flow_end"]), {k: t.data_ptr() for k, t in ts.items()})
    d.keepalive = ts
    return d


def main():
    out_dir = sys.argv[1]
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dist.init_process_group("gloo")
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    from theia_b200.engine import TadEngine, TadError

    def engine():
        uid = [TadEngine.get_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, src=0)
        return TadEngine(device=local, world_size=world, rank=rank, nccl_unique_id=uid[0])

    def everyone(x):
        got = [None] * world
        dist.all_gather_object(got, x)
        return got

    def run(eng, table, budget, name, device=False, algo="EWMA", save=True, cancel_first=False):
        eng.set_memory_budget(budget)
        mine = sharding.shard_rows(table, rank, world)
        cols = device_cols(mine) if device else eng.columns_from_numpy(mine)
        if cancel_first and rank == 0:
            job = eng.submit(cols, algo=algo, tad_id="mpasses", emit_all=True)
            job.cancel()
            dist.barrier()
        else:
            if cancel_first:
                dist.barrier()
            job = eng.submit(cols, algo=algo, tad_id="mpasses", emit_all=True)
        try:
            st = job.wait(check=False)
            st.pop("phase_ms")
            st["budget"] = budget
            if st["state"] == "COMPLETED":
                st.update(job.memory())
                st["progress"] = job.progress()
                if save:
                    np.savez(os.path.join(out_dir, "res_%s_%d.npz" % (name, rank)), **job.result())
            with open(os.path.join(out_dir, "st_%s_%d.json" % (name, rank)), "w") as fh:
                json.dump(st, fh)
            return st
        finally:
            job.release()
            cols.free()

    def passes_agree(st, name, budget_of_rank=None):
        all_st = everyone(st)
        passes = {s["passes"] for s in all_st}
        assert len(passes) == 1, (name, [s["passes"] for s in all_st])
        for r, s in enumerate(all_st):
            b = budget_of_rank(r) if budget_of_rank else s["budget"]
            assert s["state"] == "COMPLETED" and s["peak_workspace_bytes"] <= b, (name, r, s)
            assert s["progress"]["passes_done"] == s["progress"]["passes"] == s["passes"], (name, r, s["progress"])
        return passes.pop()

    eng = engine()
    tables = {n: case_table(n, world) for n in ("spread", "skewed")}
    # ---- spread table: host and device input, EWMA and DBSCAN, P >= 2 and P >= 4 --------------------------------------
    for algo in ("EWMA", "DBSCAN"):
        for device in (False, True):
            tag = "spread_%s_%s" % (algo, "dev" if device else "host")
            st = run(eng, tables["spread"], 0, tag + "_ref", device, algo)
            assert st["passes"] == 1, st
            for budget, at_least in ((BUDGET_2, 2), (BUDGET_4, 4)):
                st = run(eng, tables["spread"], budget, "%s_%d" % (tag, budget >> 20), device, algo)
                p = passes_agree(st, tag)
                assert p >= at_least, (tag, budget, p)
    # ---- skewed ownership: P from the heavy owner's counts ----------------------------------------------------------------
    run(eng, tables["skewed"], 0, "skewed_ref", True)
    st = run(eng, tables["skewed"], BUDGET_4, "skewed_64", True)
    passes_agree(st, "skewed")
    owned = [s["rows_owned"] for s in everyone(st)]
    assert owned[-1] > 2 * max(owned[:-1]), owned
    # ---- unequal budgets: the same P everywhere ------------------------------------------------------------------------
    unequal = lambda r: BUDGET_4 if r == 0 else ROOMY   # noqa: E731
    st = run(eng, tables["spread"], unequal(rank), "unequal", True)
    planned = passes_agree(st, "unequal", unequal)
    assert planned >= 4, planned
    # ---- a budget at which one rank's spill scratch does not fit: an agreed split -------------------------------------
    # one bucket per rank: every owned row takes the oversized-bucket path, whose scratch the planner does not size, so
    # rank 0's passes do not fit and every rank splits them
    eng.close()
    os.environ["TAD_DEBUG_LOGB"] = str((world - 1).bit_length())
    eng = engine()
    st = run(eng, tables["spread"], unequal(rank), "split", True)
    split_passes = passes_agree(st, "split", unequal)
    assert split_passes > planned, (split_passes, planned)
    assert st["spill_rows"] > 0
    eng.close()
    del os.environ["TAD_DEBUG_LOGB"]
    # ---- the NCCL all-to-all exchange inside the passes, chunked: the chunk count comes from the pass's largest shard --
    os.environ["TAD_PEER_PULL"] = "0"
    os.environ["TAD_EXCHANGE_MIN_ROWS"] = str(len(sharding.shard_rows(tables["spread"], 0, world)["value"]) // 8)
    eng = engine()
    st = run(eng, tables["spread"], BUDGET_4, "nccl", True)
    assert passes_agree(st, "nccl") >= 4
    eng.close()
    del os.environ["TAD_PEER_PULL"], os.environ["TAD_EXCHANGE_MIN_ROWS"]
    eng = engine()
    # ---- ARIMA in passes equals its one-pass run --------------------------------------------------------------------
    t = synth.torch_cols_to_numpy(synth.make_flows_torch(20000 * world, 40, seed=88, device=torch.device("cuda", local),
                                                         noisy=True))
    run(eng, t, 0, "arima_ref", True, "ARIMA")
    st = run(eng, t, BUDGET_4, "arima_64", True, "ARIMA")
    assert passes_agree(st, "arima") >= 2
    # ---- one rank's job cancelled right after submit: every rank's job fails CANCELLED; the contexts go on ---------
    st = run(eng, tables["spread"], BUDGET_4, "cancel", True, cancel_first=True)
    verdicts = everyone((st["state"], st["error"]))
    assert all(v == ("FAILED", -6) for v in verdicts), verdicts
    small = case_table("small", world)
    st = run(eng, small, BUDGET_4, "after_cancel", True)
    passes_agree(st, "after_cancel")
    # ---- a 1/64 range that does not fit: every rank fails NOMEM; the contexts go on ------------------------------------
    st = run(eng, case_table("one_big", world), BUDGET_4, "nomem", True, save=False)
    verdicts = everyone((st["state"], st["error"]))
    assert all(v == ("FAILED", -3) for v in verdicts), verdicts
    assert all("bytes" in m and "rank" in m for m in everyone(st["err_msg"])), st["err_msg"]
    st = run(eng, small, BUDGET_4, "after_nomem", False)
    passes_agree(st, "after_nomem")
    # ---- below the floor ---------------------------------------------------------------------------------------------
    try:
        eng.set_memory_budget(BUDGET_4 - 1)
        raise AssertionError("a budget below the floor was accepted")
    except TadError as e:
        assert e.code == -1, e
    eng.close()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
