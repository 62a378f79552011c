"""TAD_FLAG_FIT_BESIDE (an ARIMA job fits beside a running fit): the header define and the binding's flag bit, no GPU
needed."""
import os
import shutil
import subprocess

from theia_b200 import _lib
from theia_b200.engine import TadEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _spec(**kw):
    args = dict(algo="ARIMA", reducer=_lib.TAD_REDUCE_MAX, start_time=0, end_time=0, tad_id="x", emit_all=False,
                ns_ignore=(), global_rows=0, keep=[])
    args.update(kw)
    return TadEngine._spec(**args)


def test_binding_sets_the_fit_beside_bit():
    assert _lib.TAD_FLAG_FIT_BESIDE == 8
    assert _spec().flags == 0
    assert _spec(fit_beside=True).flags == _lib.TAD_FLAG_FIT_BESIDE
    assert _spec(fit_beside=True, emit_all=True).flags == _lib.TAD_FLAG_FIT_BESIDE | _lib.TAD_FLAG_EMIT_ALL


def test_submit_passes_fit_beside_through():
    import inspect
    assert inspect.signature(TadEngine.submit).parameters["fit_beside"].default is False


def test_header_define_compiles_as_c99_and_cxx17(tmp_path):
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
    src = tmp_path / "flag.c"
    src.write_text('#include "theia_tad.h"\n'
                   "_Static_assert(TAD_FLAG_FIT_BESIDE == 8u, \"TAD_FLAG_FIT_BESIDE\");\n"
                   "_Static_assert((TAD_FLAG_FIT_BESIDE & (TAD_FLAG_EMIT_ALL | TAD_FLAG_PROFILE | TAD_FLAG_SHARE)) == 0,"
                   " \"distinct bits\");\n"
                   "_Static_assert(TAD_ABI_VERSION == 2, \"ABI version\");\n"
                   "unsigned flags(void) { return TAD_FLAG_FIT_BESIDE | TAD_FLAG_EMIT_ALL; }\n")
    inc = os.path.join(ROOT, "include")
    subprocess.check_call([gcc, "-std=c99", "-pedantic", "-Wall", "-Werror", "-fsyntax-only", "-I", inc, "-x", "c",
                           str(src)])
    cxx = tmp_path / "flag.cc"
    cxx.write_text(src.read_text().replace("_Static_assert", "static_assert"))
    subprocess.check_call([gxx, "-std=c++17", "-Wall", "-Werror", "-fsyntax-only", "-I", inc, "-x", "c++", str(cxx)])
