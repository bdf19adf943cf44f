"""Host-only checks of DECIMAL columns wider than 18 digits: plan analysis accepts precision 19..38 and refuses 39 and every
construct the device does not evaluate on such values; the generated plans compile with NVRTC for sm_90a; the fixture
writer lays values out as the reference's Uncompressed encoder does (enc/Uncompressed.scala:330-345)."""
import ctypes as C
import os
import struct

import pytest

from snappydata_b200 import build
from snappydata_b200.column_format import SqlType as T, decimal_bytes, encode_wide_decimal, parse_unsafe_row, unsafe_row
from snappydata_b200.capi import Op
from snappydata_b200.plan import PlanBuilder


def _codegen(desc):
    lib = C.CDLL(build.build_codegen_lib())
    lib.sd_plan_codegen.restype = C.c_int
    lib.sd_plan_codegen.argtypes = [C.c_void_p, C.c_char_p, C.c_int64, C.POINTER(C.c_int64), C.c_char_p, C.c_int64, C.c_char_p,
                                    C.c_int64, C.c_int32, C.c_int32, C.c_int32]
    src, sig, name, ln = C.create_string_buffer(1 << 18), C.create_string_buffer(1 << 16), C.create_string_buffer(256), C.c_int64()
    rc = lib.sd_plan_codegen(C.byref(desc.c), src, len(src), C.byref(ln), sig, len(sig), name, len(name), 0, 0, 0)
    return rc, src.value.decode(errors="replace"), name.value.decode()


def _agg_plan(p, s=2):
    b = PlanBuilder()
    d, k = b.col(T.DECIMAL, 0, True, scale=s, precision=p), b.col(T.STRING, 1, False)
    b.filter(d >= b.lit(T.DECIMAL, p, s))
    b.group_by(k)
    b.sum(d).avg(d).min(d).max(d).count(d)
    return b.build()


@pytest.mark.parametrize("p", [19, 28, 38])
def test_precision_19_to_38_accepted(p):
    rc, src, _ = _codegen(_agg_plan(p))
    assert rc == 0, src
    assert "sd::dec_rec" in src


def test_precision_39_refused():
    rc, msg, _ = _codegen(_agg_plan(39))
    assert rc == 1, msg


def _refused(make):
    b = PlanBuilder()
    d = b.col(T.DECIMAL, 0, False, scale=4, precision=30)
    make(b, d)
    desc = b.build()
    for e in desc._exprs[: len(desc.exprs_py)]:   # the builder leaves an arithmetic node's (precision, scale) at 0
        if e.op == Op.ADD:
            e.c = (30 << 8) | 4
    rc, msg, _ = _codegen(desc)
    return rc, msg


@pytest.mark.parametrize("label,make", [
    ("arithmetic", lambda b, d: b.sum(d + d)),
    ("negation", lambda b, d: b.sum(-d)),
    ("cast to double", lambda b, d: b.sum(d.cast(T.DOUBLE))),
    ("cast to a narrower decimal", lambda b, d: b.sum(d.cast(T.DECIMAL, 18, 4))),
    ("cast down in scale", lambda b, d: b.sum(d.cast(T.DECIMAL, 38, 2))),
    ("startswith", lambda b, d: b.filter(d.startswith(b.lit(T.DECIMAL, 30, 4))).count()),
    ("update SET value", lambda b, d: b.update({0: d})),
])
def test_refused_constructs(label, make):
    rc, msg = _refused(make)
    assert rc == 2, (label, msg)


def test_cast_up_from_narrow_accepted():
    b = PlanBuilder()
    d, n = b.col(T.DECIMAL, 0, False, scale=4, precision=30), b.col(T.DECIMAL, 1, True, scale=2, precision=12)
    b.filter(d > n.cast(T.DECIMAL, 30, 4))
    b.max(d)
    rc, msg, _ = _codegen(b.build())
    assert rc == 0, msg


def test_wide_plans_compile_with_nvrtc():
    nvrtc = pytest.importorskip("cuda.bindings.nvrtc")
    b = PlanBuilder()   # hash keys (wide, string), wide IN list, projection of a wide column in a second plan
    d, k = b.col(T.DECIMAL, 0, True, scale=5, precision=35), b.col(T.STRING, 1, False)
    b.filter(d.isin(3) | (d < b.lit(T.DECIMAL, 10, 2).cast(T.DECIMAL, 35, 5)))
    b.group_by(d, k)
    b.sum(d).min(d).max(d).avg(d)
    pb = PlanBuilder()
    pd = pb.col(T.DECIMAL, 0, True, scale=5, precision=35)
    pb.project(pd)
    csrc = os.path.join(os.path.dirname(build.__file__), "csrc")
    hdrs = [open(os.path.join(csrc, n)).read().encode() for n in ("sd_device.h", "sd_kernels.cuh")]
    for desc in (_agg_plan(38, 18), b.build(), pb.build()):
        rc, source, name = _codegen(desc)
        assert rc == 0, source
        err, prog = nvrtc.nvrtcCreateProgram(('#include "sd_kernels.cuh"\n' + source).encode(), b"plan.cu", 2, hdrs,
                                             [b"sd_device.h", b"sd_kernels.cuh"])
        nvrtc.nvrtcAddNameExpression(prog, ("sd::scan_aggregate_kernel<%s>" % name).encode())
        opts = [b"--gpu-architecture=sm_90a", b"-std=c++17", b"--fmad=false", b"-default-device", b"-device-int128"]
        (err,) = nvrtc.nvrtcCompileProgram(prog, len(opts), opts)
        if int(err) != 0:
            _, n = nvrtc.nvrtcGetProgramLogSize(prog)
            log = b" " * n
            nvrtc.nvrtcGetProgramLog(prog, log)
            raise AssertionError(log.decode(errors="replace")[-3000:])
        nvrtc.nvrtcDestroyProgram(prog)


def test_fixture_bytes():
    assert [decimal_bytes(v).hex() for v in (0, -1, 127, 128, -129, 10 ** 38 - 1)] == \
        ["00", "ff", "7f", "0080", "ff7f", "4b3b4ca85a86c47a098a223fffffffff"]
    buf = encode_wide_decimal([128, None, -1], nulls=[False, True, False])
    assert buf == (struct.pack("<ii", 0, 8) + struct.pack("<Q", 0b010) + struct.pack("<i", 2) + b"\x00\x80" +
                   struct.pack("<i", 1) + b"\xff")
    t = (T.DECIMAL, 38, 18)
    row = unsafe_row([(t, -129), (T.INT, 5), (t, None)])
    assert parse_unsafe_row(row, [t, T.INT, t]) == [-129, 5, None]


# ---- host merges of wide-DECIMAL partial rows (sd_final_merge / sd_partial_merge; no device needed) -----------------------
def _merge_plan():
    b = PlanBuilder()
    d = b.col(T.DECIMAL, 0, True, scale=18, precision=38)
    b.sum(d).avg(d)
    return b.build()


def _partials(desc, sums):
    """partial rows [sum, avg sum, avg count] with the given totals (one row per partition)"""
    schema = desc.partial_schema()
    out = b""
    for v in sums:
        row = unsafe_row(list(zip(schema, [v, v, 1])))
        out += struct.pack("<q", len(row)) + row
    return out


def _final(sums):
    from snappydata_b200 import capi
    api, desc = capi.product_api(), _merge_plan()
    return capi.final_merge(api, desc, _partials(desc, sums))


def test_wide_sum_merges_are_exact_and_overflow_is_sticky():
    big = 9 * 10 ** 37
    assert _final([big, 5])[0][0] == big + 5
    assert _final([10 ** 20, 3 * 10 ** 20 + 1]) == [[4 * 10 ** 20 + 1, 2 * 10 ** 24 + 5000]]   # AVG at scale 22, HALF_UP
    # partial totals whose running sum passes 10^38 (and 2^127) but whose total is in range: exact, as in one execution
    assert _final([big, big, -big])[0][0] == big
    assert _final([big, big, big, -big, -big, -big, 7])[0][0] == 7
    # a total of more than 38 digits is NULL, however the rows were split
    assert _final([big, big]) == [[None, None]]
    assert _final([10 ** 38 - 1, 10 ** 38 - 1, 10 ** 38 - 1]) == [[None, None]]
    # a partition that overflowed on its own stays NULL whatever the other partitions add
    assert _final([10 ** 38, 5]) == [[None, None]]
    assert _final([10 ** 38, -big]) == [[None, None]]


def test_wide_sum_partial_merge_carries_overflow():
    from snappydata_b200 import capi
    from snappydata_b200.column_format import parse_row_stream
    api, desc = capi.product_api(), _merge_plan()
    merged = capi.partial_merge_raw(api, desc, _partials(desc, [9 * 10 ** 37, 9 * 10 ** 37]))
    rows = parse_row_stream(merged, desc.partial_schema())
    assert rows[0][0] == 10 ** 38   # the overflowed state: a total no in-range sum reaches
    assert capi.final_merge(api, desc, merged + _partials(desc, [-9 * 10 ** 37])) == [[None, None]]
