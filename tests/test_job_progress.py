"""tad_job_progress (include/theia_tad.h) without a GPU: the layout the bindings rely on and the rejected NULL arguments."""
import ctypes

from theia_b200 import _lib

TAD_ERR_INVALID_ARG = -1


def test_progress_struct_size():
    assert ctypes.sizeof(_lib.TadProgress) == 2 * 4 + 2 * 8


def test_job_progress_rejects_null_arguments():
    L = _lib.load()
    p = _lib.TadProgress(7, 7, 7, 7)
    assert L.tad_job_progress(None, ctypes.byref(p)) == TAD_ERR_INVALID_ARG
    assert (p.passes_done, p.passes, p.fits_done, p.fits_total) == (7, 7, 7, 7)        # untouched
    # a NULL output is rejected before the job is looked at, so any non-NULL handle will do
    not_a_job = ctypes.create_string_buffer(256)
    assert L.tad_job_progress(ctypes.cast(not_a_job, ctypes.c_void_p), None) == TAD_ERR_INVALID_ARG
