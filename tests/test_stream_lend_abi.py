"""TAD_FLAG_LEND (a streamed job lends the GPU while it waits for its caller): the header define, the binding's flag bit
and tad_job_lent's argument check, no GPU needed."""
import ctypes as C
import os
import shutil
import subprocess

from theia_b200 import _lib
from theia_b200.engine import TadEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAD_ERR_INVALID_ARG = -1


def _spec(**kw):
    args = dict(algo="EWMA", reducer=_lib.TAD_REDUCE_MAX, start_time=0, end_time=0, tad_id="x", emit_all=False,
                ns_ignore=(), global_rows=0, keep=[])
    args.update(kw)
    return TadEngine._spec(**args)


def test_binding_sets_the_lend_bit():
    assert _lib.TAD_FLAG_LEND == 16
    others = (_lib.TAD_FLAG_EMIT_ALL, _lib.TAD_FLAG_PROFILE, _lib.TAD_FLAG_SHARE, _lib.TAD_FLAG_FIT_BESIDE)
    assert all(_lib.TAD_FLAG_LEND & f == 0 for f in others)
    assert _spec().flags == 0
    assert _spec(lend=True).flags == _lib.TAD_FLAG_LEND
    assert _spec(lend=True, share=True).flags == _lib.TAD_FLAG_LEND | _lib.TAD_FLAG_SHARE
    assert _spec(lend=True, emit_all=True, fit_beside=True).flags == \
        _lib.TAD_FLAG_LEND | _lib.TAD_FLAG_EMIT_ALL | _lib.TAD_FLAG_FIT_BESIDE


def test_header_define_compiles_as_c99_and_cxx17(tmp_path):
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
    src = tmp_path / "lend.c"
    src.write_text('#include "theia_tad.h"\n'
                   "_Static_assert(TAD_FLAG_LEND == 16u, \"TAD_FLAG_LEND\");\n"
                   "_Static_assert((TAD_FLAG_LEND & (TAD_FLAG_EMIT_ALL | TAD_FLAG_PROFILE | TAD_FLAG_SHARE | "
                   "TAD_FLAG_FIT_BESIDE)) == 0, \"distinct bits\");\n"
                   "_Static_assert(TAD_ABI_VERSION == 2, \"ABI version\");\n"
                   "int lent(tad_job *j) { uint32_t n; double ms; return tad_job_lent(j, &n, &ms); }\n"
                   "unsigned flags(void) { return TAD_FLAG_LEND | TAD_FLAG_SHARE; }\n")
    inc = os.path.join(ROOT, "include")
    subprocess.check_call([gcc, "-std=c99", "-pedantic", "-Wall", "-Werror", "-fsyntax-only", "-I", inc, "-x", "c",
                           str(src)])
    cxx = tmp_path / "lend.cc"
    cxx.write_text(src.read_text().replace("_Static_assert", "static_assert"))
    subprocess.check_call([gxx, "-std=c++17", "-Wall", "-Werror", "-fsyntax-only", "-I", inc, "-x", "c++", str(cxx)])


def test_job_lent_rejects_null_arguments():
    L = _lib.load()
    n, ms = C.c_uint32(7), C.c_double(1.5)
    assert L.tad_job_lent(None, C.byref(n), C.byref(ms)) == TAD_ERR_INVALID_ARG
    assert L.tad_job_lent(None, None, None) == TAD_ERR_INVALID_ARG
    assert (n.value, ms.value) == (7, 1.5)
