"""Jobs streamed to every rank on several GPUs (tests/multi_stream_worker.py, one process per rank): the union of the
ranks' rows equals the oracle's bit for bit in one pass and in passes, the ranks agree on the passes and every *again,
and an omitted block or a cancel fails every rank alike, after which the contexts run the next job."""
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
def test_streamed_ranks_match_the_oracle(tmp_path, world):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    from tests.multi_passes_worker import BUDGET_4, case_table
    from tests.util import assert_same_rows, oracle_rows
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(29670 + world),
           os.path.join(ROOT, "tests", "multi_stream_worker.py"), str(tmp_path)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    spread = case_table("spread", world)
    for algo in ("EWMA", "DBSCAN"):
        want, _, _ = oracle_rows(spread, algo, emit_all=True)
        for budget in (0, BUDGET_4):
            name = "%s_%d" % (algo, budget >> 20)
            assert_same_rows(_union(tmp_path, name, world), want, what="%d ranks streamed %s" % (world, name))
    small = case_table("small", world)
    want, _, _ = oracle_rows(small, "EWMA", emit_all=True)
    assert_same_rows(_union(tmp_path, "after", world), want, what="%d ranks after the verdicts" % world)
