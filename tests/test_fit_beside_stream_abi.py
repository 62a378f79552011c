"""A streamed ARIMA job fitting beside a running fit (TAD_FLAG_SHARE | TAD_FLAG_FIT_BESIDE on tad_submit_stream): the
binding's flag bits and the header, no GPU needed."""
import inspect
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


def test_submit_stream_fit_beside_defaults_to_false():
    params = inspect.signature(TadEngine.submit_stream).parameters
    assert params["fit_beside"].default is False
    assert params["share"].default is False


def test_spec_sets_both_bits():
    assert _spec(share=True, fit_beside=True).flags == _lib.TAD_FLAG_SHARE | _lib.TAD_FLAG_FIT_BESIDE
    assert _spec(share=True).flags == _lib.TAD_FLAG_SHARE
    assert _spec(fit_beside=True).flags == _lib.TAD_FLAG_FIT_BESIDE


def test_submit_stream_passes_both_flags_to_spec(monkeypatch):
    """submit_stream hands `share` and `fit_beside` to _spec (the flags the C call receives)."""
    seen, original = {}, TadEngine._spec

    def spec(*args, **kw):
        seen["flags"] = original(*args, **kw).flags
        raise RuntimeError("stop before the C call")

    monkeypatch.setattr(TadEngine, "_spec", staticmethod(spec))
    eng = TadEngine.__new__(TadEngine)
    try:
        eng.submit_stream(algo="ARIMA", share=True, fit_beside=True)
    except RuntimeError:
        pass
    assert seen["flags"] == _lib.TAD_FLAG_SHARE | _lib.TAD_FLAG_FIT_BESIDE


def test_header_compiles_as_c99_and_cxx17(tmp_path):
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
    src = tmp_path / "flags.c"
    src.write_text('#include "theia_tad.h"\n'
                   "_Static_assert((TAD_FLAG_SHARE | TAD_FLAG_FIT_BESIDE) == 12u, \"both flags\");\n"
                   "_Static_assert(TAD_ABI_VERSION == 2, \"ABI version\");\n"
                   "int submit(tad_ctx *ctx, tad_job **out) {\n"
                   "    tad_job_spec spec = {0};\n"
                   "    spec.algo = TAD_ALGO_ARIMA;\n"
                   "    spec.flags = TAD_FLAG_SHARE | TAD_FLAG_FIT_BESIDE;\n"
                   "    return tad_submit_stream(ctx, &spec, 0, out);\n"
                   "}\n")
    inc = os.path.join(ROOT, "include")
    subprocess.check_call([gcc, "-std=c99", "-pedantic", "-Wall", "-Werror", "-fsyntax-only", "-I", inc, "-x", "c",
                           str(src)])
    cxx = tmp_path / "flags.cc"
    cxx.write_text(src.read_text().replace("_Static_assert", "static_assert").replace("= {0}", "{}"))
    subprocess.check_call([gxx, "-std=c++17", "-Wall", "-Werror", "-fsyntax-only", "-I", inc, "-x", "c++", str(cxx)])
