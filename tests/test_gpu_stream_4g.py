"""A streamed job of more than 2^32 rows on one H100: only each pass must stay below 2^32-2 rows.  Its own module, so
that no other context of the test session holds device memory when it starts."""
import time

import numpy as np
import pytest

from oracle import tad_oracle
from theia_b200 import synth

pytestmark = pytest.mark.gpu

COPIES = 65


def test_more_than_2_32_rows_per_round():
    """One device-resident block of ~6.7e7 rows (src_ip, flow_end, value) pushed 65 times per round, copy k with
    src_ip ^= k: ~4.4e9 rows per round.  The base block's src_ip values have their low 7 bits zero, so every copy is a
    set of connections of its own, and the job's result rows are the base block's result rows relabelled for every k.
    DBSCAN flags only the rare isolated spikes here, which keeps 65 copies of the result small in host memory.
    The job runs twice: with the exact hint (P = 8 from the start), and without a hint, where the first round is one
    pass whose 64-bit cursor counts all ~4.4e9 rows.  No per-residue count comes near 2^32 (that takes 64 x 2^32 rows),
    and on these paths a wrapped 32-bit cursor would not change a result either: P grows whenever a pass exceeds the
    cap, so the test checks that more than 2^32 rows per round run end to end, not the counter width by itself."""
    import torch
    from theia_b200.engine import DeviceColumns, TadEngine
    torch.cuda.empty_cache()
    if torch.cuda.mem_get_info()[0] < 60e9:
        pytest.skip("needs ~60 GB of free HBM")
    dev = torch.device("cuda", 0)
    S, n = 670_000, 100
    R = S * n
    g = torch.Generator(device=dev).manual_seed(91)
    idx = torch.arange(R, device=dev, dtype=torch.int64)
    src = ((idx // n) << 7).to(torch.int32)
    flow_end = (synth.T0 + 3600 + 60 * (idx % n)).to(torch.int32)
    value = 4_000_000_000 + torch.randint(0, 1_000_000, (R,), device=dev, generator=g)
    value += (torch.rand(R, device=dev, generator=g) < 0.001).to(torch.int64) * 40_000_000_000
    del idx
    bufs = [torch.empty_like(src), torch.empty_like(src)]
    torch.cuda.synchronize()
    torch.cuda.empty_cache()               # the default budget is what is free on the device

    def block(s):
        return DeviceColumns(R, {"src_ip": s.data_ptr(), "flow_end": flow_end.data_ptr(), "value": value.data_ptr()})

    with TadEngine(device=0) as e:
        job = e.submit(block(src), algo="DBSCAN", tad_id="base")
        base_st = job.wait()
        base = job.result()
        job.release()

        def run(hint):
            t0 = time.perf_counter()
            job = e.submit_stream(algo="DBSCAN", rows_hint=hint, tad_id="4g")
            rounds, again = 0, True
            while again:
                for k in range(COPIES):
                    b = bufs[k & 1]                 # free again: the push of copy k-1 has returned
                    torch.bitwise_xor(src, k, out=b)
                    torch.cuda.synchronize()
                    job.push(block(b))
                again = job.end()
                rounds += 1
            st = job.wait()
            wall = time.perf_counter() - t0
            mem = job.memory()
            got = job.result()
            job.release()
            print("DBSCAN, streamed %d rows per round, hint %d: %.1f s wall, %d rounds, %d passes, peak workspace %.1f GB, "
                  "device %.0f ms" % (COPIES * R, hint, wall, rounds, mem["passes"], mem["peak_workspace_bytes"] / 1e9,
                                      st["device_ms"]))
            return got, st, mem, rounds

        got, st, mem, rounds = run(COPIES * R)
        got0, st0, mem0, rounds0 = run(0)
    assert COPIES * R > 1 << 32
    assert st["rows_in"] == st["rows_kept"] == COPIES * R
    for k in ("points", "series", "result_rows"):
        assert st[k] == COPIES * base_st[k], k
    assert rounds == mem["passes"] >= 2
    assert rounds0 <= rounds + 1
    for k in ("rows_in", "rows_kept", "points", "series", "result_rows"):
        assert st0[k] == st[k], k
    want = {c: np.concatenate([base[c] ^ np.uint32(k) if c == "src_ip" else base[c] for k in range(COPIES)])
            for c in base}
    want = tad_oracle.canonicalize(want)
    for res in (got, got0):
        res = tad_oracle.canonicalize(res)
        for c in want:
            assert np.array_equal(res[c], want[c], equal_nan=True), c
