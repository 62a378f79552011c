"""TAD_FLAG_RANK_STREAM (this rank's part of a job streamed to every rank): the header define and the binding's flag bit,
no GPU needed."""
import os
import re
import shutil
import subprocess

from theia_b200 import _lib
from theia_b200.engine import TadEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "theia_tad.h")


def _spec(**kw):
    args = dict(algo="EWMA", reducer=_lib.TAD_REDUCE_MAX, start_time=0, end_time=0, tad_id="x", emit_all=False,
                ns_ignore=(), global_rows=0, keep=[])
    args.update(kw)
    return TadEngine._spec(**args)


def test_header_define_is_32_and_overlaps_no_flag():
    flags = dict(re.findall(r"#define (TAD_FLAG_\w+)\s+(\d+)u", open(HEADER).read()))
    assert int(flags.pop("TAD_FLAG_RANK_STREAM")) == 32 == _lib.TAD_FLAG_RANK_STREAM
    assert flags and all(int(v) & 32 == 0 for v in flags.values()), flags


def test_submit_stream_ranks_sets_exactly_the_bit():
    assert _spec().flags == 0
    assert _spec(ranks=True).flags == _lib.TAD_FLAG_RANK_STREAM
    assert _spec(ranks=True, emit_all=True).flags == _lib.TAD_FLAG_RANK_STREAM | _lib.TAD_FLAG_EMIT_ALL
    assert _spec(share=True, fit_beside=True, lend=True).flags & _lib.TAD_FLAG_RANK_STREAM == 0


def test_header_define_compiles_as_c99_and_cxx17(tmp_path):
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else shutil.which("gcc")
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
    src = tmp_path / "rank_stream.c"
    src.write_text('#include "theia_tad.h"\n'
                   "_Static_assert(TAD_FLAG_RANK_STREAM == 32u, \"TAD_FLAG_RANK_STREAM\");\n"
                   "_Static_assert((TAD_FLAG_RANK_STREAM & (TAD_FLAG_EMIT_ALL | TAD_FLAG_PROFILE | TAD_FLAG_SHARE | "
                   "TAD_FLAG_FIT_BESIDE | TAD_FLAG_LEND)) == 0, \"distinct bits\");\n"
                   "_Static_assert(TAD_ABI_VERSION == 2, \"ABI version\");\n"
                   "int part(tad_ctx *c, tad_job **j) {\n"
                   "    tad_job_spec s = {0};\n"
                   "    s.flags = TAD_FLAG_RANK_STREAM | TAD_FLAG_EMIT_ALL;\n"
                   "    return tad_submit_stream(c, &s, 0, j);\n"
                   "}\n")
    inc = os.path.join(ROOT, "include")
    subprocess.check_call([gcc, "-std=c99", "-pedantic", "-Wall", "-Werror", "-fsyntax-only", "-I", inc, "-x", "c",
                           str(src)])
    cxx = tmp_path / "rank_stream.cc"
    cxx.write_text(src.read_text().replace("_Static_assert", "static_assert").replace("= {0}", "= {}"))
    subprocess.check_call([gxx, "-std=c++17", "-Wall", "-Werror", "-fsyntax-only", "-I", inc, "-x", "c++", str(cxx)])
