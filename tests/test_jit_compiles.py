"""Host-only check of the NVRTC path: the generated plan struct + the kernel template compile for sm_90a for the
plan shapes the engine distinguishes (no-key / dense groups / hash table / projection; nullable columns; string
predicates) in every kernel variant (staged paths only | + per-row decode, delta and delete paths; literals
non-null | NULL literal).  NVRTC needs no GPU, so template errors in variants that only the JIT instantiates are
caught here, and the compile latency of the default variant -- the plan-compile cost a query pays once, like the
reference's Janino compile of its WholeStageCodegen class (ColumnTableScan.scala:186-672) -- is bounded."""
import ctypes as C
import os
import time

import pytest

from snappydata_b200 import build, plan as P
from snappydata_b200.column_format import SqlType as T
from snappydata_b200.plan import PlanBuilder

nvrtc = pytest.importorskip("cuda.bindings.nvrtc")


def _plans():
    out = {"c1": P.c1_plan(), "q6": P.q6_plan(), "q1": P.q1_plan()}
    b = PlanBuilder()   # integer + nullable keys -> device hash table; every aggregate function
    k, d, v, s = b.col(T.INT, 0, True), b.col(T.DATE, 1, False), b.col(T.DOUBLE, 2, True), b.col(T.STRING, 3, True)
    b.filter((d >= b.lit(T.DATE)) & s.is_not_null())
    b.group_by(k, d)
    b.count().sum(v).avg(v).min(v).max(k).count(v)
    out["hash"] = b.build()
    b = PlanBuilder()   # filter + projection, nullable columns, string equality through the dictionary
    c0, c1, c2 = b.col(T.INT, 0, True), b.col(T.DOUBLE, 1, True), b.col(T.STRING, 2, False)
    b.filter((c0 >= b.lit(T.INT)) & (c0 <= b.lit(T.INT)) & c2.eq(b.lit(T.STRING)))
    b.project(c0, c1, c2)
    out["project"] = b.build()
    b = PlanBuilder()   # nullable string key (dense table with a NULL group), boolean / short / float columns
    s, f, h, bo = b.col(T.STRING, 0, True), b.col(T.FLOAT, 1, True), b.col(T.SHORT, 2, False), b.col(T.BOOLEAN, 3, True)
    b.filter(bo | (h > b.lit(T.SHORT)))
    b.group_by(s)
    b.count().sum(f).max(h)
    out["groups_nullable"] = b.build()
    b = PlanBuilder()   # DECIMAL aggregates (two-slot wide sums), Spark casts incl. overflow-to-NULL
    dc, ic, sk = b.col(T.DECIMAL, 0, True, scale=5, precision=12), b.col(T.INT, 1, False), b.col(T.STRING, 2, True)
    b.filter(ic.cast(T.BOOLEAN) & (dc >= b.lit(T.DECIMAL, 12, 5)))
    b.group_by(sk)
    b.sum(dc).avg(dc).min(dc).sum(dc.cast(T.DOUBLE)).sum(ic.cast(T.DECIMAL, 9, 2)).sum(dc.cast(T.DECIMAL, 15, 7))
    out["decimal"] = b.build()
    b = PlanBuilder()   # raw-string predicates (byte compares), string keys by reference in the hash table, MIN / MAX(STRING)
    s1, s2, v = b.col(T.STRING, 0, True), b.col(T.STRING, 1, False), b.col(T.INT, 2, False)
    b.filter((s1 >= b.lit(T.STRING)) & s2.startswith(b.lit(T.STRING)) | s1.isin(2))
    b.group_by(s2, v)
    b.min(s1).max(s1).count()
    out["strings"] = b.build()
    b = PlanBuilder()   # 32 grouping keys of mixed types (one NULL bit each), hash table; the plan halves its tile or drops the ring
    ks = [b.col((T.INT, T.LONG, T.DATE, T.STRING)[i % 4], i, i % 3 == 0) for i in range(32)]
    v = b.col(T.DOUBLE, 32, True)
    b.group_by(*ks)
    b.count().sum(v).max(ks[1])
    out["keys32"] = b.build()
    b = PlanBuilder()   # projection of every field width (device row writer's kinds), nullable columns, raw + dictionary strings
    ts = [T.BOOLEAN, T.BYTE, T.SHORT, T.INT, T.DATE, T.FLOAT, T.DOUBLE, T.LONG, T.TIMESTAMP, T.STRING, T.DECIMAL]
    cs = [b.col(t, i, i % 2 == 0, scale=2 if t == T.DECIMAL else 0, precision=12 if t == T.DECIMAL else 0) for i, t in enumerate(ts)]
    b.filter(cs[3].is_null() | (cs[3] > b.lit(T.INT)) & cs[9].startswith(b.lit(T.STRING)))
    b.project(*cs, cs[3] + cs[2].cast(T.INT), cs[6] * cs[6])
    out["project_all"] = b.build()
    return out


def _codegen(desc, slow, litnull):
    lib = C.CDLL(build.build_codegen_lib())
    lib.sd_plan_codegen.restype = C.c_int
    lib.sd_plan_codegen.argtypes = [C.c_void_p, C.c_char_p, C.c_int64, C.POINTER(C.c_int64), C.c_char_p, C.c_int64, C.c_char_p,
                                    C.c_int64, C.c_int32, C.c_int32, C.c_int32]
    src, sig, name, ln = C.create_string_buffer(1 << 18), C.create_string_buffer(1 << 16), C.create_string_buffer(256), C.c_int64()
    rc = lib.sd_plan_codegen(C.byref(desc.c), src, len(src), C.byref(ln), sig, len(sig), name, len(name), 0, litnull, slow)
    assert rc == 0, src.value.decode(errors="replace")
    return src.value.decode(), sig.value.decode(), name.value.decode()


def _compile(source, name):
    csrc = os.path.join(os.path.dirname(build.__file__), "csrc")
    hdrs = [open(os.path.join(csrc, n)).read().encode() for n in ("sd_device.h", "sd_kernels.cuh")]
    err, prog = nvrtc.nvrtcCreateProgram(('#include "sd_kernels.cuh"\n' + source).encode(), b"plan.cu", 2, hdrs,
                                         [b"sd_device.h", b"sd_kernels.cuh"])
    assert int(err) == 0
    nvrtc.nvrtcAddNameExpression(prog, ("sd::scan_aggregate_kernel<%s>" % name).encode())
    opts = [b"--gpu-architecture=sm_90a", b"-std=c++17", b"--fmad=false", b"-default-device"]   # sd_jit.cpp's options
    t = time.time()
    (err,) = nvrtc.nvrtcCompileProgram(prog, len(opts), opts)
    dt = time.time() - t
    if int(err) != 0:
        _, n = nvrtc.nvrtcGetProgramLogSize(prog)
        log = b" " * n
        nvrtc.nvrtcGetProgramLog(prog, log)
        raise AssertionError("NVRTC failed for %s:\n%s" % (name, log.decode(errors="replace")[-3000:]))
    _, n = nvrtc.nvrtcGetCUBINSize(prog)
    assert n > 0
    nvrtc.nvrtcDestroyProgram(prog)
    return dt


@pytest.mark.parametrize("label", ["c1", "q6", "q1", "hash", "project", "groups_nullable", "decimal", "strings", "keys32", "project_all"])
def test_every_kernel_variant_compiles_for_sm_100a(label):
    # the name is the test's historical id; it compiles with sd_jit.cpp's current options, i.e. for sm_90a
    desc = _plans()[label]
    seen = set()
    for slow, litnull in ((0, 0), (1, 0), (0, 1), (1, 1)):
        source, sig, name = _codegen(desc, slow, litnull)
        assert f";slow={slow}" in sig and f";litnull={litnull}" in sig
        assert name not in seen, "variants must not share a struct name (the registry is keyed by signature)"
        seen.add(name)
        assert ("SLOW_PATHS = true" in source) == bool(slow)
        dt = _compile(source, name)
        if not slow and not litnull:
            # plan-compile latency of the variant a query normally runs (0.3-0.7 s on this image's host)
            assert dt < 8.0, f"default variant of {label} took {dt:.1f} s to compile"
