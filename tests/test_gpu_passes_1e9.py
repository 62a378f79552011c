"""A job larger than device memory on one H100, with no memory budget set: it runs in hash-range passes by itself.
Its own module, so that no other context of the test session holds device memory when it starts."""
import numpy as np
import pytest

from theia_b200 import synth
from tests.util import assert_same_rows, oracle_rows

pytestmark = pytest.mark.gpu


def _mem_available():
    try:
        for line in open("/proc/meminfo"):
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    except OSError:
        pass
    return 0


def test_beyond_device_memory_runs_in_passes():
    """BASELINE configs[2] shape (1e9 records / 1e7 connections x 100), EWMA, host-resident pinned columns, no budget:
    more than one H100 holds at once, so the job runs in passes by itself."""
    import time

    import torch
    from theia_b200.engine import TadEngine
    if _mem_available() < 64e9:
        pytest.skip("needs ~64 GB of available host memory")
    torch.cuda.empty_cache()
    if torch.cuda.mem_get_info()[0] < 70e9:
        pytest.skip("needs ~70 GB of free HBM")
    S, n = 10_000_000, 100
    R = S * n
    with TadEngine(device=0) as e:
        cols = e.alloc_columns(R)
        try:
            synth.fill_columns_blocks(cols, S, n, seed=71, device=torch.device("cuda", 0))
            torch.cuda.empty_cache()
            t0 = time.perf_counter()
            job = e.submit(cols, algo="EWMA", tad_id="1e9")
            st = job.wait()
            wall = time.perf_counter() - t0
            mem = job.memory()
            res = job.result()
            job.release()
            print("1e9-row EWMA host job: %.1f s wall, %d passes, peak workspace %.1f GB, device %.0f ms, phases %s" % (
                wall, mem["passes"], mem["peak_workspace_bytes"] / 1e9, st["device_ms"], st["phase_ms"]))
            assert mem["passes"] >= 2
            assert st["rows_in"] == R and st["points"] == R
            assert abs(int(st["series"]) - S) <= 2
            # ~3000 sampled connections against the oracle: source ips with ip % 3331 == 7
            src = cols.view("src_ip")[:R]
            mask = (src % np.uint32(3331)) == 7
            sub = {k: cols.view(k)[:R][mask].copy() for k in synth.COLUMN_DTYPES}
            want, ns, _ = oracle_rows(sub, "EWMA")
            assert ns >= 2500
            sel = (res["src_ip"] % np.uint32(3331)) == 7
            assert_same_rows({k: v[sel] for k, v in res.items()}, want, what="1e9 rows, sampled connections")
        finally:
            cols.free()
