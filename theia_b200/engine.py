"""Python host over the C ABI: the calls the reference-side shim makes, in the order it makes them.

    eng = TadEngine(device=0)
    cols = eng.columns_from_numpy(table)          # fill library-owned pinned buffers
    job = eng.submit(cols, algo="EWMA", tad_id=...)   # non-blocking, like CreateSparkApplication
    st = job.wait()                               # or poll(): state / completed_stages / total_stages
    rows = job.result()                           # dict of numpy arrays (tadetector columns)
    job.release(); cols.free(); eng.close()

Streamed input (the table arrives block by block and is never held whole):

    res, st = eng.run_stream(lambda: read_blocks(), algo="EWMA", rows_hint=n)   # re-reads while another pass needs it
    eng.set_host_budget(4 << 30)    # or keep the rows in pinned host memory between passes: read once
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib as L

_COLS = (("src_ip", np.uint32), ("dst_ip", np.uint32), ("src_port", np.uint16), ("dst_port", np.uint16),
         ("proto", np.uint8), ("flow_start", np.uint32), ("flow_end", np.uint32), ("value", np.uint64))
_NS_COLS = (("src_ns", np.uint32), ("dst_ns", np.uint32))
_OUT = (("src_ip", np.uint32), ("dst_ip", np.uint32), ("src_port", np.uint16), ("dst_port", np.uint16),
        ("proto", np.uint8), ("flow_start", np.uint32), ("flow_end", np.uint32), ("stddev", np.float64),
        ("algo_calc", np.float64), ("throughput", np.float64), ("anomaly", np.uint8))


class TadError(RuntimeError):
    def __init__(self, code, msg=""):
        self.code = code
        name = L.load().tad_strerror(code).decode()
        super().__init__("%s (%d)%s" % (name, code, (": " + msg) if msg else ""))


def _status_dict(st: L.TadStatus) -> dict:
    d = {k: getattr(st, k) for k in ("completed_stages", "total_stages", "error", "rows_in", "rows_kept", "rows_owned",
                                     "points", "series", "result_rows", "spill_rows", "gpu_launches", "device_ms",
                                     "total_ms")}
    d["state"] = L.STATE_NAMES[st.state]
    d["err_msg"] = st.err_msg.decode(errors="replace")
    d["phase_ms"] = {n: st.phase_ms[i] for i, n in enumerate(L.PHASE_NAMES)}
    return d


class Columns:
    """Library-owned pinned-host (or device) column buffers (tad_alloc_columns)."""

    def __init__(self, eng: "TadEngine", capacity: int, mem: int = L.TAD_MEM_HOST):
        self.eng = eng
        self.c = L.TadColumns()
        rc = eng.lib.tad_alloc_columns(eng.ctx, capacity, mem, C.byref(self.c))
        if rc != 0:
            raise TadError(rc, "tad_alloc_columns(%d)" % capacity)
        self.owned = True

    def view(self, name: str) -> np.ndarray:
        """numpy view of a host column (capacity elements)."""
        assert self.c.mem == L.TAD_MEM_HOST
        dt = dict(_COLS + _NS_COLS)[name]
        n = int(self.c.capacity)
        ptr = getattr(self.c, name)
        buf = (C.c_char * (n * np.dtype(dt).itemsize)).from_address(ptr)
        return np.frombuffer(buf, dtype=dt, count=n)

    def fill(self, table: dict):
        n = len(table["flow_end"])
        assert n <= self.c.capacity
        for name, dt in _COLS:
            a = table.get(name)
            if a is None:
                self.view(name)[:n] = 0
            else:
                self.view(name)[:n] = np.asarray(a, dtype=dt)
        if table.get("src_ns") is not None or table.get("dst_ns") is not None:
            rc = self.eng.lib.tad_alloc_ns_columns(self.eng.ctx, C.byref(self.c))
            if rc != 0:
                raise TadError(rc, "tad_alloc_ns_columns")
            for name, dt in _NS_COLS:
                a = table.get(name)
                self.view(name)[:n] = 0 if a is None else np.asarray(a, dtype=dt)
        self.c.rows = n
        return self

    def free(self):
        if self.owned and self.c.capacity:
            self.eng.lib.tad_free_columns(self.eng.ctx, C.byref(self.c))
            self.owned = False


class DeviceColumns:
    """Columns that already live in HBM (raw device pointers, e.g. torch tensors' data_ptr())."""

    def __init__(self, rows: int, ptrs: dict):
        self.c = L.TadColumns()
        self.c.rows = rows
        self.c.capacity = rows
        self.c.mem = L.TAD_MEM_DEVICE
        for name, _ in _COLS:
            setattr(self.c, name, ptrs.get(name))
        self.keepalive = ptrs

    def free(self):
        pass


class Job:
    def __init__(self, eng, handle, keep):
        self.eng = eng
        self.h = handle
        self._keep = keep

    def poll(self) -> dict:
        st = L.TadStatus()
        self.eng.lib.tad_poll(self.h, C.byref(st))
        return _status_dict(st)

    def wait(self, timeout_ms: int = -1, check: bool = True) -> dict:
        st = L.TadStatus()
        self.eng.lib.tad_wait(self.h, timeout_ms, C.byref(st))
        d = _status_dict(st)
        if check and d["state"] == "FAILED":
            raise TadError(st.error, d["err_msg"])
        return d

    def result(self, copy: bool = True) -> dict:
        r = L.TadRows()
        rc = self.eng.lib.tad_result(self.h, C.byref(r))
        if rc != 0:
            raise TadError(rc, "tad_result")
        n = int(r.rows)
        out = {}
        for name, dt in _OUT:
            if n == 0:
                out[name] = np.zeros(0, dtype=dt)
                continue
            buf = (C.c_char * (n * np.dtype(dt).itemsize)).from_address(getattr(r, name))
            a = np.frombuffer(buf, dtype=dt, count=n)
            out[name] = a.copy() if copy else a
        return out

    def memory(self) -> dict:
        """Of a COMPLETED job: the hash-range passes it ran in, the largest device workspace the context held, the rows
        that went through the host row store and the most store bytes the context held."""
        passes, peak = C.c_uint32(), C.c_uint64()
        rc = self.eng.lib.tad_job_memory(self.h, C.byref(passes), C.byref(peak))
        if rc != 0:
            raise TadError(rc, "tad_job_memory")
        stored, peak_host = C.c_uint64(), C.c_uint64()
        rc = self.eng.lib.tad_job_host_memory(self.h, C.byref(stored), C.byref(peak_host))
        if rc != 0:
            raise TadError(rc, "tad_job_host_memory")
        return {"passes": passes.value, "peak_workspace_bytes": peak.value, "stored_rows": stored.value,
                "peak_host_bytes": peak_host.value}

    def progress(self) -> dict:
        """In any state (tad_job_progress): the hash-range passes finished and planned so far, and the ARIMA prefix fits
        finished and those of the passes whose fit phase has started (0 / 0 for the other algorithms)."""
        p = L.TadProgress()
        rc = self.eng.lib.tad_job_progress(self.h, C.byref(p))
        if rc != 0:
            raise TadError(rc, "tad_job_progress")
        return {"passes_done": p.passes_done, "passes": p.passes, "fits_done": p.fits_done, "fits_total": p.fits_total}

    def yields(self) -> dict:
        """Of a COMPLETED ARIMA job (tad_job_yields): how many times its fit phase yielded to queued jobs and the time
        it was parked meanwhile (see TadEngine.set_fit_sharing)."""
        n, ms = C.c_uint32(), C.c_double()
        rc = self.eng.lib.tad_job_yields(self.h, C.byref(n), C.byref(ms))
        if rc != 0:
            raise TadError(rc, "tad_job_yields")
        return {"yields": n.value, "parked_ms": ms.value}

    def lent(self) -> dict:
        """Of a COMPLETED streamed job (tad_job_lent): the number of queued jobs that ran while it lent the GPU waiting
        for its caller, and the time it was lent (see TadEngine.submit_stream's ``lend``)."""
        n, ms = C.c_uint32(), C.c_double()
        rc = self.eng.lib.tad_job_lent(self.h, C.byref(n), C.byref(ms))
        if rc != 0:
            raise TadError(rc, "tad_job_lent")
        return {"jobs_run": n.value, "lent_ms": ms.value}

    def cancel(self):
        """tad_cancel: returns at once; an ARIMA job on one GPU stops within one evaluation round of its fit kernel."""
        self.eng.lib.tad_cancel(self.h)

    def release(self):
        if self.h:
            self.eng.lib.tad_release(self.h)
            self.h = None


def _block_columns(block):
    """(TadColumns, objects to keep alive) of one streamed block: a numpy dict (any host memory; a missing or None
    column is NULL), Columns or DeviceColumns."""
    if isinstance(block, (Columns, DeviceColumns)):
        return block.c, block
    c = L.TadColumns()
    n = len(block["flow_end"])
    c.rows = c.capacity = n
    c.mem = L.TAD_MEM_HOST
    keep = []
    for name, dt in _COLS + _NS_COLS:
        a = block.get(name)
        if a is None:
            continue
        a = np.ascontiguousarray(a, dtype=dt)
        if len(a) != n:
            raise ValueError("column %s has %d values, flow_end has %d" % (name, len(a), n))
        keep.append(a)
        setattr(c, name, a.ctypes.data if n else C.addressof(_EMPTY))
    return c, keep


_EMPTY = C.c_uint64(0)     # a non-NULL address for the columns of an empty numpy block
_TEXT_SLOTS = ("src_ip", "dst_ip", "src_ns", "dst_ns")


class StreamJob(Job):
    """A job fed with column blocks (tad_submit_stream): push() every block of a round, then end(); while end() returns
    True the engine needs the same rows once more."""

    def __init__(self, eng, handle, keep):
        super().__init__(eng, handle, keep)
        self._last = None

    def push(self, block, text=None):
        """``text``: {"src_ip" / "dst_ip" / "src_ns" / "dst_ns": (column bytes, marks)} -- those slots as Native String
        column bytes with the byte offset of every 32nd row (tad_stream_push_text_ns).  The address slots are encoded
        into job-wide ids on the GPU; the namespace slots are tested there against the ignore list given as names
        (submit_stream's ``ns_ignore_names``)."""
        c, keep = _block_columns(block)
        if text:
            tx = []
            for slot in _TEXT_SLOTS:
                if slot not in text:
                    tx.append(None)
                    continue
                data, marks = text[slot]
                data = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data
                marks = np.ascontiguousarray(marks, dtype=np.uint64)
                t = L.TadTextColumn()
                t.bytes = data.ctypes.data if len(data) else C.addressof(_EMPTY)
                t.nbytes = len(data)
                t.marks = marks.ctypes.data if len(marks) else C.addressof(_EMPTY)
                keep = [keep, data, marks]
                tx.append(t)
            keep = [keep, tx]
            rc = self.eng.lib.tad_stream_push_text_ns(self.h, C.byref(c), *(C.byref(t) if t is not None else None for t in tx))
        else:
            rc = self.eng.lib.tad_stream_push(self.h, C.byref(c))
        if rc != 0:
            raise TadError(rc, self.poll()["err_msg"])
        self._last = (c, keep)        # the engine may read this block until the next push or end returns

    def names(self, slot: str):
        """Of a COMPLETED job: the dictionary of a text slot as numpy (bytes, offsets): id k is bytes[offsets[k]:offsets[k+1]]."""
        b, o, n = C.c_void_p(), C.c_void_p(), C.c_uint32()
        rc = self.eng.lib.tad_job_names(self.h, ("src_ip", "dst_ip").index(slot), C.byref(b), C.byref(o), C.byref(n))
        if rc != 0:
            raise TadError(rc, "tad_job_names")
        offsets = np.ctypeslib.as_array((C.c_uint64 * (n.value + 1)).from_address(o.value)).copy()
        nbytes = int(offsets[-1])
        data = np.frombuffer((C.c_char * nbytes).from_address(b.value), dtype=np.uint8).copy() if nbytes else \
            np.zeros(0, dtype=np.uint8)
        return data, offsets

    def end(self) -> bool:
        again = C.c_int32()
        rc = self.eng.lib.tad_stream_end(self.h, C.byref(again))
        if rc != 0:
            raise TadError(rc, self.poll()["err_msg"])
        self._last = None
        return bool(again.value)


class TadEngine:
    def __init__(self, device: int = 0, world_size: int = 1, rank: int = 0, nccl_unique_id: bytes | None = None,
                 memory_budget: int | None = None, host_budget: int | None = None):
        self.lib = L.load()
        cfg = L.TadConfig()
        cfg.device, cfg.world_size, cfg.rank = device, world_size, rank
        self._uid = None
        if nccl_unique_id is not None:
            self._uid = C.create_string_buffer(bytes(nccl_unique_id), 128)
            cfg.nccl_unique_id = C.cast(self._uid, C.c_void_p)
            cfg.nccl_unique_id_bytes = 128
        ctx = C.c_void_p()
        rc = self.lib.tad_init(C.byref(cfg), C.byref(ctx))
        if rc != 0:
            raise TadError(rc, "tad_init(device=%d)" % device)
        self.ctx = ctx
        if memory_budget is not None:
            self.set_memory_budget(memory_budget)
        if host_budget is not None:
            self.set_host_budget(host_budget)

    def set_host_budget(self, nbytes: int):
        """Pinned host bytes the context may hold for its host row store (0 = none): a streamed job that needs several
        passes then keeps its rows there and is delivered once."""
        rc = self.lib.tad_set_host_budget(self.ctx, int(nbytes))
        if rc != 0:
            raise TadError(rc, "tad_set_host_budget(%d)" % nbytes)

    def set_memory_budget(self, nbytes: int):
        """Device bytes the context's workspace may hold; larger jobs run in passes.  0 = free memory at job start on one
        GPU, no planning on a rank engine (world_size > 1), where every rank of a job must set a budget or none."""
        rc = self.lib.tad_set_memory_budget(self.ctx, int(nbytes))
        if rc != 0:
            raise TadError(rc, "tad_set_memory_budget(%d)" % nbytes)

    def set_fit_sharing(self, reserve: int):
        """Single GPU (tad_set_fit_sharing): with a nonzero reserve (at least 64 MiB) an ARIMA job's fit phase yields to
        queued EWMA and DBSCAN jobs, which run in the reserve while it is parked; the ARIMA job plans in the memory
        budget less the reserve.  Streamed jobs take part when submitted with ``share=True``.  0 (default) = off: jobs
        run in submit order."""
        rc = self.lib.tad_set_fit_sharing(self.ctx, int(reserve))
        if rc != 0:
            raise TadError(rc, "tad_set_fit_sharing(%d)" % reserve)

    @staticmethod
    def get_unique_id() -> bytes:
        buf = C.create_string_buffer(128)
        rc = L.load().tad_get_unique_id(buf, 128)
        if rc != 0:
            raise TadError(rc, "tad_get_unique_id")
        return buf.raw

    @staticmethod
    def loopback_id(world_size: int) -> bytes:
        """A 128-byte id for ``world_size`` rank engines on ONE device in this process (tad_debug_loopback_id): passed
        as their ``nccl_unique_id``, they talk through an in-process loopback instead of NCCL and CUDA IPC, and take
        turns on the device.  For tests of the multi-rank paths on a single GPU.  Once the ranks are created (or their
        creation failed), release_loopback_id(id) drops it, so that no context joins it later and an id not every rank
        joined is not kept for the life of the process."""
        buf = C.create_string_buffer(128)
        rc = L.load().tad_debug_loopback_id(int(world_size), buf, 128)
        if rc != 0:
            raise TadError(-1, "tad_debug_loopback_id(%d)" % world_size)
        return buf.raw

    @staticmethod
    def release_loopback_id(uid: bytes):
        """tad_debug_loopback_release: the ranks that joined keep their group; no further context may join it."""
        buf = C.create_string_buffer(bytes(uid), 128)
        if L.load().tad_debug_loopback_release(buf, 128) != 0:
            raise TadError(-1, "tad_debug_loopback_release")

    def alloc_columns(self, capacity: int, mem: int = L.TAD_MEM_HOST) -> Columns:
        return Columns(self, capacity, mem)

    def columns_from_numpy(self, table: dict) -> Columns:
        return self.alloc_columns(max(1, len(table["flow_end"]))).fill(table)

    @staticmethod
    def _spec(algo, reducer, start_time, end_time, tad_id, emit_all, ns_ignore, global_rows, keep, share=False,
              fit_beside=False, lend=False, ranks=False):
        spec = L.TadJobSpec()
        spec.algo = L.ALGOS[algo] if isinstance(algo, str) else int(algo)
        spec.reducer = reducer
        spec.start_time, spec.end_time = int(start_time), int(end_time)
        spec.flags = (L.TAD_FLAG_EMIT_ALL if emit_all else 0) | (L.TAD_FLAG_SHARE if share else 0) | \
            (L.TAD_FLAG_FIT_BESIDE if fit_beside else 0) | (L.TAD_FLAG_LEND if lend else 0) | \
            (L.TAD_FLAG_RANK_STREAM if ranks else 0)
        spec.id = tad_id.encode()[:39]
        spec.global_rows = int(global_rows)
        if len(ns_ignore):
            arr = np.asarray(ns_ignore, dtype=np.uint32)
            spec.n_ns_ignore = len(arr)
            spec.ns_ignore = arr.ctypes.data
            keep.append(arr)
        return spec

    def _checked(self, job, rc, check):
        if rc != 0 and check:
            msg = job.poll()["err_msg"] if job.h else ""
            job.release()
            raise TadError(rc, msg)
        return job

    def submit(self, cols, algo="EWMA", reducer: int = L.TAD_REDUCE_MAX, start_time: int = 0, end_time: int = 0,
               tad_id: str = "", emit_all: bool = False, ns_ignore=(), check: bool = True, global_rows: int = 0,
               fit_beside: bool = False) -> Job:
        """``fit_beside``: TAD_FLAG_FIT_BESIDE, an ARIMA job queued behind another ARIMA job's fit may fit beside it
        while fit sharing is on (set_fit_sharing), instead of waiting for the whole fit phase."""
        keep = [cols]
        spec = self._spec(algo, reducer, start_time, end_time, tad_id, emit_all, ns_ignore, global_rows, keep,
                          fit_beside=fit_beside)
        h = C.c_void_p()
        rc = self.lib.tad_submit(self.ctx, C.byref(spec), C.byref(cols.c), C.byref(h))
        return self._checked(Job(self, h, keep), rc, check)

    def submit_stream(self, algo="EWMA", reducer: int = L.TAD_REDUCE_MAX, start_time: int = 0, end_time: int = 0,
                      ns_ignore=(), rows_hint: int = 0, emit_all: bool = False, tad_id: str = "",
                      check: bool = True, text_filter=None, share: bool = False,
                      fit_beside: bool = False, ns_ignore_names=None, lend: bool = False,
                      ranks: bool = False) -> StreamJob:
        """A job whose rows arrive as blocks (tad_submit_stream); ``rows_hint``: one round's rows, 0 = unknown.
        ``text_filter``: row predicates evaluated on the GPU (tad_submit_stream_filtered): {"src_ip" / "dst_ip":
        (op, pattern bytes) with op one of "any", "eq", "nonempty", "icontains", "proto_eq": 0..255}; absent keys hold
        for every row.  ``share``: TAD_FLAG_SHARE, the job takes part in fit sharing (set_fit_sharing): an ARIMA job's
        fit yields, an EWMA or DBSCAN job may run while a fit is parked.  ``fit_beside``: TAD_FLAG_FIT_BESIDE, with
        ``share`` an ARIMA job queued behind another ARIMA job's fit may fit beside it once its first block is pushed.
        ``ns_ignore_names``: the namespace ignore list as names (bytes), for a job that pushes its namespace columns as
        text (tad_submit_stream_filtered_ns); ``ns_ignore`` (ids) is then empty.  ``lend``: TAD_FLAG_LEND, while fit
        sharing is on the job plans in the budget less the reserve and, while it waits for the next block, runs queued
        EWMA and DBSCAN submit() jobs in the reserve (StreamJob.lent()).  ``ranks``: TAD_FLAG_RANK_STREAM, on a rank
        engine (world_size > 1) the job is this rank's part of a job streamed to every rank: each rank's caller pushes
        any disjoint share of the rows, ``rows_hint`` is this rank's share; ignored on one GPU."""
        keep = []
        spec = self._spec(algo, reducer, start_time, end_time, tad_id, emit_all, ns_ignore, 0, keep, share, fit_beside,
                          lend, ranks)
        h = C.c_void_p()
        if text_filter is None and ns_ignore_names is None:
            rc = self.lib.tad_submit_stream(self.ctx, C.byref(spec), int(rows_hint), C.byref(h))
        else:
            text_filter = text_filter or {}
            flt = L.TadStreamFilter()
            for t, slot in enumerate(("src_ip", "dst_ip")):
                op, pat = text_filter.get(slot, ("any", b""))
                flt.op[t] = L.TAD_NAME_OPS[op] if isinstance(op, str) else int(op)
                pat = bytes(pat)
                buf = C.create_string_buffer(pat, len(pat) or 1)
                keep.append(buf)
                flt.pattern[t] = C.cast(buf, C.c_void_p).value
                flt.pattern_len[t] = len(pat)
            flt.proto_eq = int(text_filter.get("proto_eq", -1))
            if ns_ignore_names is None:
                rc = self.lib.tad_submit_stream_filtered(self.ctx, C.byref(spec), int(rows_hint), C.byref(flt), C.byref(h))
            else:
                names = [bytes(x) for x in ns_ignore_names]
                data = np.frombuffer(b"".join(names) or b"\0", dtype=np.uint8)
                off = np.zeros(len(names) + 1, dtype=np.uint64)
                off[1:] = np.cumsum([len(x) for x in names], dtype=np.uint64)
                keep += [data, off]
                fns = L.TadStreamFilterNs(flt, len(names), data.ctypes.data, off.ctypes.data)
                rc = self.lib.tad_submit_stream_filtered_ns(self.ctx, C.byref(spec), int(rows_hint), C.byref(fns),
                                                            C.byref(h))
        return self._checked(StreamJob(self, h, keep), rc, check)

    def run(self, table: dict, on_job=None, memory_budget: int | None = None, **kw):
        """Convenience: numpy table in, (result dict, status dict) out.  ``on_job(job)`` is called right after tad_submit
        (the caller may poll it from another thread) and ``on_job(None)`` before the handle is released.
        ``memory_budget``: set the context's budget (tad_set_memory_budget) before the job; the status then carries
        ``memory`` = Job.memory()."""
        if memory_budget is not None:
            self.set_memory_budget(memory_budget)
        cols = self.columns_from_numpy(table)
        job = self.submit(cols, **kw)
        if on_job is not None:
            on_job(job)
        try:
            st = job.wait()
            if memory_budget is not None:
                st["memory"] = job.memory()
            return job.result(), st
        finally:
            if on_job is not None:
                on_job(None)
            job.release()
            cols.free()

    def run_stream(self, blocks_factory, memory_budget: int | None = None, **kw):
        """Convenience: ``blocks_factory()`` yields one round's blocks (numpy dicts, Columns or DeviceColumns); it is
        called once per round while the engine asks for the rows again.  Returns (result dict, status dict) like run();
        the status also carries ``rounds`` and ``memory`` = Job.memory()."""
        if memory_budget is not None:
            self.set_memory_budget(memory_budget)
        job = self.submit_stream(**kw)
        try:
            rounds, again = 0, True
            while again:
                for block in blocks_factory():
                    job.push(block)
                again = job.end()
                rounds += 1
            st = job.wait()
            st["rounds"] = rounds
            st["memory"] = job.memory()
            return job.result(), st
        finally:
            job.release()

    def close(self):
        if self.ctx:
            self.lib.tad_shutdown(self.ctx)
            self.ctx = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()
