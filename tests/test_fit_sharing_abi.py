"""tad_set_fit_sharing / tad_job_yields argument and state checks that need no GPU."""
import ctypes as C

from theia_b200 import _lib

TAD_ERR_INVALID_ARG = -1
TAD_ERR_STATE = -5
MB = 1 << 20


def test_null_context_is_rejected():
    """Without a GPU no context exists; the floor on a real context is checked in test_gpu_fit_sharing.py."""
    L = _lib.load()
    assert L.tad_set_fit_sharing(None, 0) == TAD_ERR_INVALID_ARG
    assert L.tad_set_fit_sharing(None, 64 * MB) == TAD_ERR_INVALID_ARG
    assert L.tad_set_fit_sharing(None, 1) == TAD_ERR_INVALID_ARG


def test_null_job_is_rejected():
    L = _lib.load()
    n, ms = C.c_uint32(7), C.c_double(1.5)
    assert L.tad_job_yields(None, C.byref(n), C.byref(ms)) == TAD_ERR_INVALID_ARG
    assert (n.value, ms.value) == (7, 1.5)


def test_failed_job_has_no_yields():
    """tad_job_yields answers TAD_ERR_STATE for a job that has not COMPLETED; without a GPU the one such job there is is
    an invalid submit, which tad_submit returns FAILED before it queues it on the context (an invalid job is never
    retried), so a placeholder context handle stands in and is never used."""
    L = _lib.load()
    spec = _lib.TadJobSpec()
    spec.algo = 99                                   # not an algorithm: the job is returned FAILED at once
    cols = _lib.TadColumns()
    h = C.c_void_p()
    rc = L.tad_submit(C.c_void_p(1), C.byref(spec), C.byref(cols), C.byref(h))
    assert rc == TAD_ERR_INVALID_ARG and h.value
    try:
        n = C.c_uint32(7)
        assert L.tad_job_yields(h, C.byref(n), None) == TAD_ERR_STATE
        assert n.value == 7
    finally:
        L.tad_release(h)
