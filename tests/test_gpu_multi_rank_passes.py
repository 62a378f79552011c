"""Multi-GPU jobs in hash-range passes under a memory budget: the union of the ranks' rows equals the oracle's and the
same engine's no-budget run bit for bit, every rank reports the same pass count and stays inside its own budget, and a
split, a cancel or a NOMEM verdict is taken by every rank together (tests/multi_passes_worker.py, one process per rank)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _union(out_dir, name, world):
    parts = [np.load(os.path.join(out_dir, "res_%s_%d.npz" % (name, r))) for r in range(world)]
    return {k: np.concatenate([p[k] for p in parts]) for k in parts[0].files}


@pytest.mark.parametrize("world", [2, 4])
def test_passes_on_gpus_match_the_oracle(tmp_path, world):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    from tests.multi_passes_worker import BUDGET_2, BUDGET_4, case_table
    from tests.util import assert_same_rows, oracle_rows
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(29650 + world),
           os.path.join(ROOT, "tests", "multi_passes_worker.py"), str(tmp_path)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]

    spread = case_table("spread", world)
    for algo in ("EWMA", "DBSCAN"):
        want, _, _ = oracle_rows(spread, algo, emit_all=True)
        for src in ("host", "dev"):
            tag = "spread_%s_%s" % (algo, src)
            ref = _union(tmp_path, tag + "_ref", world)
            assert_same_rows(ref, want, what="%d ranks, %s, no budget vs oracle" % (world, tag))
            for budget in (BUDGET_2, BUDGET_4):
                got = _union(tmp_path, "%s_%d" % (tag, budget >> 20), world)
                assert_same_rows(got, want, what="%d ranks, %s, %d MiB vs oracle" % (world, tag, budget >> 20))
    want, _, _ = oracle_rows(spread, "EWMA", emit_all=True)
    for name in ("unequal", "split", "nccl"):
        assert_same_rows(_union(tmp_path, name, world), want, what="%d ranks, %s vs oracle" % (world, name))
    skewed = case_table("skewed", world)
    want, _, _ = oracle_rows(skewed, "EWMA", emit_all=True)
    assert_same_rows(_union(tmp_path, "skewed_ref", world), want, what="%d ranks, skewed, no budget" % world)
    assert_same_rows(_union(tmp_path, "skewed_64", world), want, what="%d ranks, skewed, 64 MiB" % world)
    # ARIMA: a series' fits do not depend on the series that share its launch, so the passes equal the one-pass run
    assert_same_rows(_union(tmp_path, "arima_64", world), _union(tmp_path, "arima_ref", world),
                     what="%d ranks, ARIMA in passes vs no budget" % world)
    # the contexts run the next job after a cancel
    small = case_table("small", world)
    want, _, _ = oracle_rows(small, "EWMA", emit_all=True)
    assert_same_rows(_union(tmp_path, "after_cancel", world), want, what="%d ranks, after a cancel" % world)
    for r in range(world):
        st = json.load(open(os.path.join(tmp_path, "st_cancel_%d.json" % r)))
        assert "cancelled" in st["err_msg"], st
