"""Parity of the hash-range pass drivers between two builds: a fixed, seeded matrix of small jobs, and per job everything a
caller can observe except times -- the tad_status counters (gpu_launches included), state and error text, tad_job_memory
and tad_job_host_memory, tad_job_progress, a streamed job's rounds and the `again` sequence tad_stream_end returned, the
text slots' dictionaries, and a SHA-256 of the result rows sorted by every column.

    python profiles/pass_parity.py --out A.json          # run the matrix with the library of this tree
    python profiles/pass_parity.py --compare A.json B.json

The matrix: every input kind (device-resident, pinned host, streamed 65,536-row blocks hinted / unhinted / over-hinted,
streamed with a host row store that holds the round and one that falls back, streamed text keys with one IPv6 address in
five, streamed with string predicates) at no budget, a two-pass budget and the 64 MiB floor; then EWMA, DBSCAN and a small
ARIMA table in passes, oversized-bucket spills under the floor, and a job cancelled while it waits behind another; then
fit sharing: an ARIMA fit that parks for a submitted EWMA job and a streamed DBSCAN job, a queued job too large for the
reserve, and a cancel of the parked ARIMA job.
Run it with each build in the same GPU session; --compare prints every difference and exits 1 if there is one."""
import argparse
import hashlib
import json
import os
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

MB = 1 << 20
TWO_PASSES = 150 * MB          # the 2M-row table runs in two passes under it
DBSCAN_TWO_PASSES = 100 * MB   # DBSCAN's one pass is smaller: it needs a lower budget for two passes or more
SHARE_BUDGET = 1024 * MB       # fit sharing: the ARIMA job plans in it less the reserve
SHARE_RESERVE = 256 * MB
BLOCK = 65536
STATUS = ("state", "error", "err_msg", "completed_stages", "total_stages", "rows_in", "rows_kept", "rows_owned", "points",
          "series", "result_rows", "spill_rows", "gpu_launches")


def rows_sha(res):
    """SHA-256 of the result rows in the order of all their columns' bit patterns."""
    import numpy as np
    names = sorted(res)
    bits = [np.ascontiguousarray(res[k]).view("u%d" % res[k].dtype.itemsize) for k in names]
    order = np.lexsort(bits[::-1]) if len(bits[0]) else np.zeros(0, dtype=np.int64)
    h = hashlib.sha256()
    for k, b in zip(names, bits):
        h.update(k.encode())
        h.update(np.ascontiguousarray(b[order]).tobytes())
    return h.hexdigest()


def varuint(n):
    out = bytearray()
    while True:
        b = n & 0x7F
        n >>= 7
        out.append(b | (0x80 if n else 0))
        if not n:
            return bytes(out)


def name_of(v):
    """The text of address value v: one IPv6 address in five, IPv4 otherwise."""
    if v % 5 == 0:
        return b"fd00::%x:%x" % (v >> 16, v & 0xFFFF)
    return b"%d.%d.%d.%d" % ((v >> 24) & 255, (v >> 16) & 255, (v >> 8) & 255, v & 255)


def text_column(values):
    """(Native String column bytes, byte offset of every 32nd row) of the names of `values`."""
    import numpy as np
    uniq, inv = np.unique(values, return_inverse=True)
    enc = [varuint(len(name_of(int(v)))) + name_of(int(v)) for v in uniq]
    lens = np.array([len(e) for e in enc], dtype=np.uint64)[inv]
    starts = np.zeros(len(inv), dtype=np.uint64)
    if len(inv) > 1:
        np.cumsum(lens[:-1], out=starts[1:])
    return b"".join(enc[i] for i in inv), starts[::32].copy()


def job_record(job, st, timed=()):
    """`timed`: status fields left out because they depend on timing (a yielding fit's resume launches)."""
    rec = {k: st[k] for k in STATUS if k not in timed}
    rec["progress"] = job.progress()
    if st["state"] == "COMPLETED":
        rec["memory"] = job.memory()
        rec["rows_sha256"] = rows_sha(job.result())
    return rec


def run_table(eng, cols, budget, **kw):
    eng.set_memory_budget(budget)
    job = eng.submit(cols, **kw)
    try:
        return job_record(job, job.wait(check=False))
    finally:
        job.release()


def stream_blocks(table, text=False):
    """The table in 65,536-row numpy blocks; with `text` the address columns go as text slots."""
    blocks = []
    for lo in range(0, len(table["flow_end"]), BLOCK):
        b = {k: v[lo:lo + BLOCK] for k, v in table.items()}
        txt = None
        if text:
            txt = {s: text_column(b[s]) for s in ("src_ip", "dst_ip")}
            b["src_ip"] = b["dst_ip"] = None
        blocks.append((b, txt))
    return blocks


def feed(job, blocks, again_seq):
    """Every round of a streamed job until its input is complete; what each tad_stream_end returned goes to again_seq."""
    again = True
    while again and len(again_seq) < 200:
        try:
            for b, txt in blocks:
                job.push(b, text=txt)
            again = job.end()
        except Exception as e:           # a failed job: its status tells why
            again_seq.append("error: %s" % e)
            break
        again_seq.append(again)


def run_stream(eng, table, budget, hint, host=0, text=False, **kw):
    """One streamed job: 65,536-row numpy blocks; with `text` the address columns go as text slots."""
    eng.set_memory_budget(budget)
    eng.set_host_budget(host)
    blocks = stream_blocks(table, text)
    job = eng.submit_stream(rows_hint=hint, **kw)
    again_seq = []
    try:
        feed(job, blocks, again_seq)
        rec = job_record(job, job.wait(check=False))
        rec["again"] = again_seq
        if text and rec["state"] == "COMPLETED":
            rec["names_sha256"] = {s: hashlib.sha256(b"".join(x.tobytes() for x in job.names(s))).hexdigest()
                                   for s in ("src_ip", "dst_ip")}
        return rec
    finally:
        job.release()
        eng.set_host_budget(0)


def wait_fitting(job, timeout=120.0):
    """Until the ARIMA job's fit phase has started (or it has ended)."""
    t0 = time.time()
    while job.progress()["fits_done"] == 0 and job.poll()["state"] in ("SCHEDULED", "RUNNING"):
        if time.time() - t0 > timeout:
            raise RuntimeError("the fit phase did not start")
        time.sleep(0.002)


def run_sharing(eng, arima, cols, table, big):
    """Fit sharing: the ARIMA job on `arima` parks its pass for queued jobs, which run in the reserve (`cols`: `table` in
    host columns; `big`: a table whose 1/64 hash range does not fit 64 MiB).  Only what does not depend on when the
    yields come is recorded: not the ARIMA job's launches, its yield count or its progress after a cancel."""
    out = {}
    blocks = stream_blocks(table)
    eng.set_memory_budget(SHARE_BUDGET)
    eng.set_fit_sharing(SHARE_RESERVE)
    try:
        # an EWMA job and a flagged streamed DBSCAN job, queued together once the fit has started, run in its yield
        job = eng.submit(arima, algo="ARIMA", emit_all=True)
        wait_fitting(job)
        ewma = eng.submit(cols, emit_all=True)
        dbscan = eng.submit_stream(algo="DBSCAN", rows_hint=len(table["flow_end"]), share=True)
        again_seq = []
        fd = threading.Thread(target=feed, args=(dbscan, blocks, again_seq))
        fd.start()
        out["share/arima"] = job_record(job, job.wait(check=False), timed=("gpu_launches",))
        out["share/arima"]["yielded"] = job.yields()["yields"] >= 1
        out["share/ewma"] = job_record(ewma, ewma.wait(check=False))
        fd.join()
        out["share/dbscan-stream"] = job_record(dbscan, dbscan.wait(check=False))
        out["share/dbscan-stream"]["again"] = again_seq
        for j in (job, ewma, dbscan):
            j.release()

        # a job too large for a 64 MiB reserve: it goes back to its place in the queue and runs after the fit
        eng.set_fit_sharing(64 * MB)
        job = eng.submit(arima, algo="ARIMA", emit_all=True)
        wait_fitting(job)
        q = eng.submit(big)
        out["share-too-large/arima"] = job_record(job, job.wait(check=False), timed=("gpu_launches",))
        out["share-too-large/arima"]["yielded"] = job.yields()["yields"] >= 1
        out["share-too-large/queued"] = job_record(q, q.wait(check=False))
        job.release()
        q.release()

        # a cancel of the parked ARIMA job: it fails once the job run in its place has ended
        eng.set_fit_sharing(SHARE_RESERVE)
        job = eng.submit(arima, algo="ARIMA", emit_all=True)
        wait_fitting(job)
        q = eng.submit(cols, emit_all=True)
        t0 = time.time()
        while q.poll()["state"] == "SCHEDULED" and time.time() - t0 < 5.0:
            time.sleep(0.001)
        job.cancel()
        st = job.wait(check=False)
        out["share-cancel/arima"] = {k: st[k] for k in ("state", "error", "err_msg")}
        out["share-cancel/in-its-place"] = job_record(q, q.wait(check=False))
        job.release()
        q.release()
    finally:
        eng.set_fit_sharing(0)
        eng.set_memory_budget(0)
    return out


def run_matrix():
    import numpy as np
    import torch
    from theia_b200 import synth
    from theia_b200.engine import DeviceColumns, TadEngine

    signed = {np.dtype(np.uint32): np.int32, np.dtype(np.uint16): np.int16, np.dtype(np.uint64): np.int64,
              np.dtype(np.uint8): np.uint8}

    def device_cols(table):
        ts = {k: torch.from_numpy(np.ascontiguousarray(v).view(signed[v.dtype])).cuda() for k, v in table.items()}
        d = DeviceColumns(len(table["flow_end"]), {k: t.data_ptr() for k, t in ts.items()})
        d.keepalive = ts
        return d

    out = {}
    t = synth.make_flows(20000, 100, seed=61)                       # 2M rows
    n = len(t["flow_end"])
    with TadEngine(device=0) as eng:
        dev = device_cols(t)
        host = eng.columns_from_numpy(t)
        for budget in (0, TWO_PASSES, 64 * MB):
            out["device/%d" % budget] = run_table(eng, dev, budget, emit_all=True)
        for budget in (0, DBSCAN_TWO_PASSES, 64 * MB):
            out["device-dbscan/%d" % budget] = run_table(eng, dev, budget, algo="DBSCAN")
        for budget in (0, TWO_PASSES, 64 * MB):
            out["host/%d" % budget] = run_table(eng, host, budget, emit_all=True)
            for name, hint in (("hinted", n), ("unhinted", 0), ("over-hinted", 4 * n)):
                out["stream-%s/%d" % (name, budget)] = run_stream(eng, t, budget, hint, emit_all=True)
            for host_budget in (1 << 30, 64 * MB):                  # a store that holds the round; one that falls back
                out["stream-store-%d/%d" % (host_budget, budget)] = run_stream(eng, t, budget, n, host=host_budget,
                                                                                emit_all=True)
            out["stream-text/%d" % budget] = run_stream(eng, t, budget, n, text=True, emit_all=True)
            out["stream-text-store/%d" % budget] = run_stream(eng, t, budget, n, host=1 << 30, text=True)
            out["stream-predicates/%d" % budget] = run_stream(
                eng, t, budget, n, text=True, emit_all=True,
                text_filter={"src_ip": ("icontains", b"fd00"), "dst_ip": ("nonempty", b"")})
        dev.free()
        host.free()

        # ---- algorithms and edge cases ----
        ns = dict(t)
        rng = np.random.default_rng(64)
        ns["src_ns"] = rng.integers(0, 6, n).astype(np.uint32)
        ns["dst_ns"] = rng.integers(0, 6, n).astype(np.uint32)
        cols = eng.columns_from_numpy(ns)
        out["host-ns-window/64M"] = run_table(eng, cols, 64 * MB, ns_ignore=(1, 4), start_time=synth.T0 + 600,
                                              end_time=synth.T0 + 3600, emit_all=True)
        cols.free()
        out["stream-ns/64M"] = run_stream(eng, ns, 64 * MB, n, ns_ignore=(1, 4), reducer=1, emit_all=True)
        a = synth.torch_cols_to_numpy(synth.make_flows_torch(2000, 40, seed=63, device=torch.device("cuda", 0), noisy=True))
        cols = eng.columns_from_numpy(a)
        for budget in (0, 64 * MB):
            out["arima/%d" % budget] = run_table(eng, cols, budget, algo="ARIMA", emit_all=True)
        cols.free()
        small, big = synth.make_flows(20000, 100, seed=65), synth.make_flows(30, 6000, seed=66)
        sp = {k: np.concatenate([small[k], big[k]]) for k in small}
        cols = eng.columns_from_numpy(sp)
        out["spill/64M"] = run_table(eng, cols, 64 * MB, emit_all=True)
        out["spill-stream/64M"] = run_stream(eng, sp, 64 * MB, len(sp["flow_end"]), emit_all=True)
        # a job cancelled while it waits in the queue behind another: the outcome does not depend on timing
        eng.set_memory_budget(64 * MB)
        first = eng.submit(cols, emit_all=True)
        second = eng.submit(cols, emit_all=True)
        second.cancel()
        out["queued-first/64M"] = job_record(first, first.wait(check=False))
        out["queued-cancelled/64M"] = job_record(second, second.wait(check=False))
        first.release()
        second.release()
        cols.free()

        # ---- fit sharing ----
        # a fit phase of about 1.4 s, long enough to be parked
        a = synth.torch_cols_to_numpy(synth.make_flows_torch(20000, 100, seed=67, device=torch.device("cuda", 0),
                                                             noisy=True))
        arima, cols = eng.columns_from_numpy(a), eng.columns_from_numpy(t)
        big_t = synth.make_flows_torch(500_000, 100, seed=31, device=torch.device("cuda", 0))    # 5e7 rows
        torch.cuda.synchronize()
        big = DeviceColumns(int(big_t["value"].numel()), {k: v.data_ptr() for k, v in big_t.items()})
        big.keepalive = big_t
        out.update(run_sharing(eng, arima, cols, t, big))
        arima.free()
        cols.free()
        big.free()
    return out


def compare(a_path, b_path):
    a, b = (json.load(open(p)) for p in (a_path, b_path))
    diffs = []
    for case in sorted(set(a) | set(b)):
        if case not in a or case not in b:
            diffs.append("%s: only in %s" % (case, a_path if case in a else b_path))
        elif a[case] != b[case]:
            for k in sorted(set(a[case]) | set(b[case])):
                if a[case].get(k) != b[case].get(k):
                    diffs.append("%s.%s: %r != %r" % (case, k, a[case].get(k), b[case].get(k)))
    for d in diffs:
        print(d)
    print(json.dumps({"cases": len(set(a) | set(b)), "differences": len(diffs)}))
    return 1 if diffs else 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="write the matrix's records here (JSON)")
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"))
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    if not args.out:
        ap.error("--out or --compare")
    rec = run_matrix()
    with open(args.out, "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
    # the matrix covers two passes only where the two-pass budget gives them
    one_pass = sorted(k for k, v in rec.items()
                      if k.endswith(("/%d" % TWO_PASSES, "dbscan/%d" % DBSCAN_TWO_PASSES))
                      and v.get("memory", {}).get("passes", 0) < 2)
    print(json.dumps({"cases": len(rec), "failed": sorted(k for k, v in rec.items() if v["state"] != "COMPLETED"),
                      "passes": {k: v.get("memory", {}).get("passes") for k, v in sorted(rec.items())},
                      "two_pass_budget_in_one_pass": one_pass}))
    if one_pass:
        sys.exit(1)


if __name__ == "__main__":
    main()
