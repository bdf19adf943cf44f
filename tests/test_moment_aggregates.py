"""Host-only checks of STDDEV / VARIANCE / SKEWNESS / KURTOSIS: Spark 2.1.1 CentralMomentAgg as tests/moments_reference.py
restates it (closed forms, edge cases), the product's host merges (sd_final_merge / sd_partial_merge) against it and against
exact Fraction arithmetic, the partial-row schemas, plan acceptance and refusal, and NVRTC compiles of moment plans."""
import ctypes as C
import math
import os
import random
import struct
from fractions import Fraction

import pytest

import moments_reference as R
from snappydata_b200 import build, capi
from snappydata_b200.capi import AggFn
from snappydata_b200.column_format import SqlType as T, parse_row_stream, unsafe_row
from snappydata_b200.plan import PlanBuilder

FNS = R.MOMENT_FNS


def _codegen(desc):
    lib = C.CDLL(build.build_codegen_lib())
    lib.sd_plan_codegen.restype = C.c_int
    lib.sd_plan_codegen.argtypes = [C.c_void_p, C.c_char_p, C.c_int64, C.POINTER(C.c_int64), C.c_char_p, C.c_int64, C.c_char_p,
                                    C.c_int64, C.c_int32, C.c_int32, C.c_int32]
    src, sig, name, ln = C.create_string_buffer(1 << 18), C.create_string_buffer(1 << 16), C.create_string_buffer(256), C.c_int64()
    rc = lib.sd_plan_codegen(C.byref(desc.c), src, len(src), C.byref(ln), sig, len(sig), name, len(name), 0, 0, 0)
    return rc, src.value.decode(errors="replace"), name.value.decode()


def _all_fns_plan(keyed=False, nullable=True):
    b = PlanBuilder()
    x = b.col(T.DOUBLE, 0, nullable)
    if keyed:
        b.group_by(b.col(T.STRING, 1, False))
    for fn in FNS:
        b.agg(fn, x)
    return b.build()


def _partials(desc, bufs_per_partition, keys=None):
    """partial rows: one per partition, the buffers of every aggregate in plan order"""
    schema = desc.partial_schema()
    out = b""
    for i, bufs in enumerate(bufs_per_partition):
        vals = ([keys[i]] if keys else []) + [v for buf in bufs for v in buf]
        row = unsafe_row(list(zip(schema, vals)))
        out += struct.pack("<q", len(row)) + row
    return out


def _bufs(xs):
    return [R.welford(xs, R.ORDER[fn]) for fn in FNS]


def _exact_bufs(xs):
    """a partition's buffers exact, rounded once: what a merge of them is measured against is the merge alone (Spark's row-order
    update itself loses about 1e-7 of sigma per row at mean 1e9)"""
    n, mean, m2, m3, m4 = R.exact_moments(xs)
    return [[float(n), float(mean), float(m2), float(m3), float(m4)][: R.ORDER[fn] + 1] for fn in FNS]


def _final(desc, parts):
    return capi.final_merge(capi.product_api(), desc, _partials(desc, [_bufs(p) for p in parts]))


def test_partial_and_final_schemas_are_sparks_buffers():
    d = _all_fns_plan(keyed=True)
    assert d.partial_schema() == [T.STRING] + [T.DOUBLE] * (3 + 3 + 3 + 3 + 4 + 5)
    assert d.final_schema() == [T.STRING] + [T.DOUBLE] * 6
    b = PlanBuilder()
    b.stddev(b.col(T.DOUBLE, 0)).variance(b.col(T.DOUBLE, 0))
    assert [fn for fn, _ in b.build().aggs_py] == [AggFn.STDDEV_SAMP, AggFn.VAR_SAMP]


@pytest.mark.parametrize("N", [2, 3, 10, 1001])
def test_closed_forms_of_1_to_N(N):
    xs = [float(i) for i in range(1, N + 1)]
    want = {AggFn.VAR_POP: (N * N - 1) / 12, AggFn.VAR_SAMP: N * (N + 1) / 12, AggFn.SKEWNESS: 0.0,
            AggFn.KURTOSIS: -6 * (N * N + 1) / (5 * (N * N - 1))}
    want[AggFn.STDDEV_POP], want[AggFn.STDDEV_SAMP] = math.sqrt(want[AggFn.VAR_POP]), math.sqrt(want[AggFn.VAR_SAMP])
    for fn in FNS:   # the reference itself, in row order
        got = R.evaluate(fn, R.welford(xs, R.ORDER[fn]))
        assert R.close(fn, got, want[fn]), (fn, got, want[fn])
    # the product's final merge over the reference's buffers of three partitions
    parts = [xs[0::3], xs[1::3], xs[2::3]]
    (row,) = _final(_all_fns_plan(), parts)
    for fn, got in zip(FNS, row):
        assert R.close(fn, got, want[fn]), (fn, got, want[fn])


def test_constant_column_gives_exact_zero_variance():
    xs = [1e9 + 0.125] * 1000
    for fn in FNS:
        assert R.evaluate(fn, R.welford(xs, R.ORDER[fn])) in (0.0,) or math.isnan(R.evaluate(fn, R.welford(xs, R.ORDER[fn])))
    (row,) = _final(_all_fns_plan(), [xs[:300], xs[300:], []])
    assert row[:4] == [0.0, 0.0, 0.0, 0.0]
    assert math.isnan(row[4]) and math.isnan(row[5])


def test_one_value_and_no_value():
    (row,) = _final(_all_fns_plan(), [[3.5]])
    got = dict(zip(FNS, row))
    assert got[AggFn.VAR_POP] == 0.0 and got[AggFn.STDDEV_POP] == 0.0
    assert math.isnan(got[AggFn.VAR_SAMP]) and math.isnan(got[AggFn.STDDEV_SAMP])
    assert math.isnan(got[AggFn.SKEWNESS]) and math.isnan(got[AggFn.KURTOSIS])
    assert _final(_all_fns_plan(), [[None, None], []]) == [[None] * 6]
    # a no-key aggregate over no partitions: one row of Spark's initial buffers, evaluated to NULL
    desc = _all_fns_plan()
    assert capi.final_merge(capi.product_api(), desc, b"") == [[None] * 6]
    merged = parse_row_stream(capi.partial_merge_raw(capi.product_api(), desc, b""), desc.partial_schema())
    assert merged == [[0.0] * len(desc.partial_schema())]


def test_nan_and_infinity_inputs_give_nan():
    for bad in (math.nan, math.inf, -math.inf):
        (row,) = _final(_all_fns_plan(), [[1.0, 2.0], [bad, 3.0]])
        assert all(math.isnan(v) for v in row), (bad, row)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_host_merge_of_split_buffers_matches_exact_arithmetic(seed):
    rng = random.Random(seed)
    centre, spread = [(0.0, 1.0), (1e9, 1.0), (0.0, 1e-6), (-5e6, 3e3)][seed % 4]
    xs = [centre + rng.gauss(0, spread) * (1 + (i % 7 == 0) * 4) for i in range(4000)]
    parts, i = [], 0
    while i < len(xs):
        k = rng.randint(1, 900)
        parts.append(xs[i:i + k])
        i += k
    parts.insert(2, [])   # a partition without rows
    desc = _all_fns_plan()
    (row,) = capi.final_merge(capi.product_api(), desc, _partials(desc, [_exact_bufs(p) for p in parts]))
    for fn, got in zip(FNS, row):
        assert R.close(fn, got, R.exact(fn, xs)), (fn, got, R.exact(fn, xs))


def test_two_rank_partial_merge_equals_one_rank():
    api, desc = capi.product_api(), _all_fns_plan(keyed=True)
    rng = random.Random(9)
    rows = [(bytes([97 + rng.randint(0, 3)]), 1e9 + rng.gauss(0, 2)) for _ in range(3000)]
    by = lambda sub: {k: [x for kk, x in sub if kk == k] for k in sorted({k for k, _ in sub})}

    def partial(sub):
        g = by(sub)
        return _partials(desc, [_exact_bufs(v) for v in g.values()], keys=list(g))
    one = capi.final_merge(api, desc, partial(rows))
    two = capi.final_merge(api, desc, capi.partial_merge_raw(api, desc, partial(rows[:1700]) + partial(rows[1700:])))
    assert sorted(r[0] for r in one) == sorted(r[0] for r in two)
    for a, b in zip(sorted(one), sorted(two)):
        for fn, x, y in zip(FNS, a[1:], b[1:]):
            assert R.close(fn, y, x), (fn, x, y)
        exact = [R.exact(fn, by(rows)[a[0]]) for fn in FNS]
        assert all(R.close(fn, g, w) for fn, g, w in zip(FNS, a[1:], exact))


def test_naive_power_sums_miss_the_bar():
    rng = random.Random(4)
    xs = [1e9 + rng.gauss(0, 1) for _ in range(10000)]
    want = R.exact(AggFn.VAR_SAMP, xs)
    assert abs(R.naive(AggFn.VAR_SAMP, xs) - want) > 1e-3 * want


@pytest.mark.parametrize("t", [T.INT, T.LONG, T.FLOAT, T.DECIMAL])
def test_non_double_input_is_refused(t):
    for fn in FNS:
        b = PlanBuilder()
        x = b.col(t, 0, False, scale=2 if t == T.DECIMAL else 0)
        b.agg(fn, x)
        rc, msg, _ = _codegen(b.build())
        assert rc == 1, (t, fn, msg)
        b = PlanBuilder()
        b.agg(fn, b.col(t, 0, False, scale=2 if t == T.DECIMAL else 0).cast(T.DOUBLE))   # Spark's implicit cast
        rc, msg, _ = _codegen(b.build())
        assert rc == 0, (t, fn, msg)


def test_moment_plans_share_shift_and_sums():
    b = PlanBuilder()
    x, y = b.col(T.DOUBLE, 0, True), b.col(T.DOUBLE, 1, False)
    b.stddev_samp(x).var_pop(x).kurtosis(x).skewness(y).avg(x)
    rc, src, _ = _codegen(b.build())
    assert rc == 0, src
    assert "NSHIFT = 2;" in src
    assert src.count("sd::shift_cand") == 2   # one shift per input, shared by its aggregates


def _plans_for_nvrtc():
    out = []
    for keyed in ("none", "dense", "hash"):
        b = PlanBuilder()
        x, q = b.col(T.DOUBLE, 0, True), b.col(T.INT, 2, False)
        b.filter(q > b.lit(T.INT))
        if keyed == "dense":
            b.group_by(b.col(T.STRING, 1, True))
        elif keyed == "hash":
            b.group_by(q)
        b.stddev_pop(x).stddev_samp(x).var_pop(x).var_samp(x).skewness(x).kurtosis(q.cast(T.DOUBLE)).count()
        out.append(b.build())
    return out


def test_moment_plans_compile_with_nvrtc():
    nvrtc = pytest.importorskip("cuda.bindings.nvrtc")
    csrc = os.path.join(os.path.dirname(build.__file__), "csrc")
    hdrs = [open(os.path.join(csrc, n)).read().encode() for n in ("sd_device.h", "sd_kernels.cuh")]
    for desc in _plans_for_nvrtc():
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


def test_exact_reference_is_exact():
    xs = [1.0, 2.0, 4.0]
    n, mean, m2, m3, m4 = R.exact_moments(xs)
    assert (n, mean, m2) == (3, Fraction(7, 3), Fraction(42, 9))
