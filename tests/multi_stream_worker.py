"""Worker of tests/test_gpu_multi_rank_stream.py: jobs streamed to every rank (TAD_FLAG_RANK_STREAM), launched with
torch.distributed.run, one process per rank.

    python -m torch.distributed.run --nproc-per-node N tests/multi_stream_worker.py <out_dir>

Every rank is dealt a random share of each table (not its owner's rows), cut into uneven host and device blocks, and
saves its result rows (res_<case>_<rank>.npz) and status (st_<case>_<rank>.json).  Checks that need every rank's view
(the same passes and *again everywhere, the same verdict everywhere) are made here."""
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.multi_passes_worker import BUDGET_4, case_table  # noqa: E402
from tests.test_gpu_loopback_stream import cut, deal  # noqa: E402


def main():
    out_dir = sys.argv[1]
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dist.init_process_group("gloo")
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    from theia_b200.engine import TadEngine, TadError
    uid = [TadEngine.get_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    eng = TadEngine(device=local, world_size=world, rank=rank, nccl_unique_id=uid[0])

    def everyone(x):
        got = [None] * world
        dist.all_gather_object(got, x)
        return got

    def run(table, name, budget, algo="EWMA", hook=None):
        eng.set_memory_budget(budget)
        share = deal(table, world, 7)[rank]
        blocks = cut(share, 31 + rank, True)
        job = eng.submit_stream(algo=algo, tad_id="mstream", emit_all=True, rows_hint=len(share["flow_end"]), ranks=True)
        agains, code, stopped = [], None, False
        try:
            rnd = 0
            while not stopped:
                for k, b in enumerate(blocks):
                    h = hook(job, rnd, k) if hook else True
                    if h == "stop":          # return without pushing or ending: the job is released below
                        stopped = True
                        break
                    if h:
                        job.push(b)
                if stopped:
                    break
                again = job.end()
                agains.append(again)
                if not again:
                    break
                rnd += 1
        except TadError as e:
            code = e.code
        if stopped:                          # a release of a job whose input has not ended cancels it on every rank
            job.release()
            st = {"state": "FAILED", "error": -6, "err_msg": "released", "agains": agains, "code": code}
            everyone(st)
            return st
        try:
            st = job.wait(check=False)
            st.pop("phase_ms")
            st.update(agains=agains, code=code)
            if st["state"] == "COMPLETED":
                st.update(job.memory())
                np.savez(os.path.join(out_dir, "res_%s_%d.npz" % (name, rank)), **job.result())
            with open(os.path.join(out_dir, "st_%s_%d.json" % (name, rank)), "w") as fh:
                json.dump(st, fh)
        finally:
            job.release()
        all_st = everyone(st)
        if st["state"] == "COMPLETED":
            assert len({s["passes"] for s in all_st}) == 1, (name, [s["passes"] for s in all_st])
            assert len({tuple(s["agains"]) for s in all_st}) == 1, (name, [s["agains"] for s in all_st])
        else:
            assert len({(s["state"], s["error"]) for s in all_st}) == 1, (name, all_st)
        return st

    spread = case_table("spread", world)
    for algo in ("EWMA", "DBSCAN"):
        for budget in (0, BUDGET_4):
            st = run(spread, "%s_%d" % (algo, budget >> 20), budget, algo)
            assert st["state"] == "COMPLETED", st
    last = len(cut(deal(spread, world, 7)[1], 32, False)) - 1
    st = run(spread, "omit", BUDGET_4, hook=lambda j, rnd, k: rank != 1 or not (rnd == 1 and k == last))
    assert (st["state"], st["error"]) == ("FAILED", -1) and "rank 1" in st["err_msg"], st

    def cancel_mid(job, rnd, k):
        if rank == 0 and rnd == 0 and k == 2:
            job.cancel()
        return True
    st = run(spread, "cancel", BUDGET_4, hook=cancel_mid)
    assert (st["state"], st["error"], st["code"]) == ("FAILED", -6, -6), st
    last = len(cut(deal(spread, world, 7)[1], 32, False)) - 1
    st = run(spread, "release", BUDGET_4, hook=lambda j, rnd, k: "stop" if rank == 1 and k == last else True)
    assert (st["state"], st["error"]) == ("FAILED", -6), st
    st = run(case_table("one_big", world), "nomem", BUDGET_4)
    assert (st["state"], st["error"]) == ("FAILED", -3) and "rank" in st["err_msg"] and "bytes" in st["err_msg"], st

    def text_push(job, rnd, k):
        if rank == 0 and k == 1:
            b = {"flow_end": np.zeros(3, np.uint32), "value": np.zeros(3, np.uint64)}
            try:
                job.push(b, text={"src_ip": (b"\x01a\x01b\x01c", np.zeros(1, np.uint64))})
            except TadError as e:
                assert e.code == -7, e
                return False                 # the later pushes and end fail once every rank has ended the round
            raise AssertionError("text key columns were accepted on a rank stream job")
        return True
    st = run(spread, "text", BUDGET_4, hook=text_push)
    assert (st["state"], st["error"]) == ("FAILED", -7), st
    st = run(case_table("small", world), "after", BUDGET_4)
    assert st["state"] == "COMPLETED", st
    eng.close()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
