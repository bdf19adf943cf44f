"""The C-ABI library loads on a box with no GPU and exports every function include/snappy_gpu.h declares
(no compute call is made).  Also checks the ctypes mirror's struct sizes against the C compiler's."""
import ctypes as C
import os
import re
import subprocess
import tempfile

from snappydata_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_functions():
    src = open(os.path.join(ROOT, "include", "snappy_gpu.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(sdx?_[a-z_0-9]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    api = capi.product_api()
    names = declared_functions()
    assert len(names) >= 25
    missing = [n for n in names if not hasattr(api.lib, n)]
    assert not missing, missing
    assert b"sm_90a" in api.version()


def test_ctypes_struct_layout_matches_the_header():
    prog = r'''
#include <stdio.h>
#include <stddef.h>
#include "snappy_gpu.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(sd_column), sizeof(sd_expr), sizeof(sd_agg), sizeof(sd_plan_desc),
         sizeof(sd_literal), sizeof(sd_batch), offsetof(sd_batch, stats_ncols), offsetof(sd_plan_desc, literal_types));
  return 0;
}'''
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "t.c")
        open(src, "w").write(prog)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    want = [C.sizeof(capi.sd_column), C.sizeof(capi.sd_expr), C.sizeof(capi.sd_agg), C.sizeof(capi.sd_plan_desc),
            C.sizeof(capi.sd_literal), C.sizeof(capi.sd_batch), capi.sd_batch.stats_ncols.offset,
            capi.sd_plan_desc.literal_types.offset]
    assert got == want


def test_no_cpu_fallback_when_library_missing(monkeypatch):
    """The product path fails loudly when the CUDA extension is missing."""
    monkeypatch.setattr(capi, "_product", None)
    monkeypatch.setattr(capi, "LIB_PATH", "/nonexistent/libsnappygpu.so")
    try:
        capi.product_api()
        assert False, "expected SdError"
    except capi.SdError as e:
        assert "no CPU fallback" in str(e)
