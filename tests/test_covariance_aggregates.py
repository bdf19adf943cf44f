"""Host-only checks of COVAR_POP / COVAR_SAMP / CORR: Spark 2.1.1 Covariance / Corr as tests/covariance_reference.py restates
them (closed forms, edge cases), the product's host merges (sd_final_merge / sd_partial_merge) against them and against exact
Fraction arithmetic, the partial-row schemas, the refusal of PAIR nodes where they do not belong, slot and shift sharing, and
NVRTC compiles of covariance plans."""
import math
import os
import random

import pytest

import covariance_reference as R
from snappydata_b200 import build, capi
from snappydata_b200.capi import AggFn, Op
from snappydata_b200.column_format import SqlType as T, parse_row_stream
from snappydata_b200.plan import E, PlanBuilder
from test_moment_aggregates import _codegen, _partials

FNS = R.PAIR_FNS


def _all_fns_plan(keyed=False, nullable=True):
    b = PlanBuilder()
    x, y = b.col(T.DOUBLE, 0, nullable), b.col(T.DOUBLE, 2, nullable)
    if keyed:
        b.group_by(b.col(T.STRING, 1, False))
    b.covar_pop(x, y).covar_samp(x, y).corr(x, y)
    return b.build()


def _bufs(rows):
    return [R.update(rows, fn == AggFn.CORR) for fn in FNS]


def _exact_bufs(rows):
    """a partition's buffers exact, rounded once: what a merge of them is measured against is the merge alone"""
    return [[float(v) for v in R.exact_buffers(rows)][: R.FIELDS[fn]] for fn in FNS]


def _final(desc, parts, bufs=_bufs):
    return capi.final_merge(capi.product_api(), desc, _partials(desc, [bufs(p) for p in parts]))


def _check(row, rows):
    scale = R.exact_scale(rows)
    for fn, got in zip(FNS, row):
        want = R.exact(fn, rows)
        assert R.close(fn, got, want, scale), (fn, got, want)


def test_partial_and_final_schemas_are_sparks_buffers():
    d = _all_fns_plan(keyed=True)
    assert d.partial_schema() == [T.STRING] + [T.DOUBLE] * (4 + 4 + 6)
    assert d.final_schema() == [T.STRING] + [T.DOUBLE] * 3
    b = PlanBuilder()
    x, y = b.col(T.DOUBLE, 0), b.col(T.DOUBLE, 1)
    b.corr(x, y)
    d = b.build()
    assert [fn for fn, _ in d.aggs_py] == [AggFn.CORR]
    node = d.aggs_py[0][1]
    assert d.exprs_py[node][0] == Op.PAIR and d.exprs_py[node][1] == T.DOUBLE


@pytest.mark.parametrize("a,c", [(3.0, 5.0), (-0.5, 1e9), (1e-6, -2.0)])
def test_closed_forms_of_a_line(a, c):
    """y = a x + c: CORR = sign(a), COVAR = a * var(x)"""
    xs = [float(i) for i in range(1, 1001)]
    rows = [(x, a * x + c) for x in xs]
    n = len(xs)
    var_pop = (n * n - 1) / 12
    want = {AggFn.COVAR_POP: a * var_pop, AggFn.COVAR_SAMP: a * var_pop * n / (n - 1), AggFn.CORR: math.copysign(1.0, a)}
    for fn in FNS:   # the reference itself, in row order (y is rounded, so only nearly the closed form)
        got = R.evaluate(fn, R.update(rows, fn == AggFn.CORR))
        assert abs(got - want[fn]) <= 1e-6 * abs(want[fn]), (fn, got, want[fn])
    parts = [rows[0::3], rows[1::3], rows[2::3]]
    (row,) = _final(_all_fns_plan(), parts)
    for fn, got in zip(FNS, row):
        assert abs(got - want[fn]) <= 1e-6 * abs(want[fn]), (fn, got, want[fn])
    (row,) = _final(_all_fns_plan(), parts, _exact_bufs)
    _check(row, rows)


def test_constant_y_gives_exact_zero_covariance():
    rows = [(1e9 + i * 0.25, 7.5) for i in range(1000)]
    (row,) = _final(_all_fns_plan(), [rows[:300], rows[300:], []])
    assert row[0] == 0.0 and row[1] == 0.0 and math.isnan(row[2])
    for fn in FNS:
        v = R.evaluate(fn, R.update(rows, fn == AggFn.CORR))
        assert v == 0.0 or (fn == AggFn.CORR and math.isnan(v))


def test_one_row_no_row_and_nulls():
    (row,) = _final(_all_fns_plan(), [[(3.5, -1.0)]])
    assert row[0] == 0.0 and math.isnan(row[1]) and math.isnan(row[2])
    # NULL in x only, in y only, in both: none of them counts
    nulls = [(None, 1.0), (2.0, None), (None, None)]
    assert R.update(nulls) == [0.0] * 6
    assert _final(_all_fns_plan(), [nulls, []]) == [[None] * 3]
    rows = [(1.0, 2.0), (None, 5.0), (2.0, 4.5), (3.0, None), (None, None), (4.0, 9.0)]
    (row,) = _final(_all_fns_plan(), [rows[:2], rows[2:]])
    _check(row, rows)
    assert R.update(rows) == R.update(R.counted(rows))
    # a no-key aggregate over no partitions: one row of Spark's initial buffers, evaluated to NULL
    desc = _all_fns_plan()
    assert capi.final_merge(capi.product_api(), desc, b"") == [[None] * 3]
    merged = parse_row_stream(capi.partial_merge_raw(capi.product_api(), desc, b""), desc.partial_schema())
    assert merged == [[0.0] * len(desc.partial_schema())]


def test_non_finite_inputs_give_nan():
    """The device writes NaN into every buffer but n of a group with a NaN / +-Inf x or y; the merges keep the results NaN."""
    def with_bad(rows):
        bufs = _bufs(rows)
        if any(not math.isfinite(v) for r in R.counted(rows) for v in r):
            bufs = [[b[0]] + [math.nan] * (len(b) - 1) for b in bufs]
        return bufs
    for bad in (math.nan, math.inf, -math.inf):
        for rows in ([(1.0, 2.0), (bad, 3.0)], [(1.0, 2.0), (3.0, bad)]):
            (row,) = _final(_all_fns_plan(), [[(5.0, 1.0), (6.0, 2.0)], rows], with_bad)
            assert all(math.isnan(v) for v in row), (bad, row)
            assert all(math.isnan(R.exact(fn, rows)) for fn in FNS)


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_host_merge_of_split_buffers_matches_exact_arithmetic(seed):
    rng = random.Random(seed)
    (cx, sx), (cy, sy), rho = [((0.0, 1.0), (0.0, 1.0), 0.9), ((1e9, 1.0), (1e9, 1.0), 0.9), ((0.0, 1e-6), (0.0, 1e-6), 0.0),
                               ((-5e6, 3e3), (2e3, 1e-2), -1.0)][seed % 4]
    rows = []
    for i in range(4000):
        z1, z2 = rng.gauss(0, 1), rng.gauss(0, 1)
        zy = -z1 if rho == -1.0 else rho * z1 + math.sqrt(1 - rho * rho) * z2
        rows.append((cx + sx * z1, cy + sy * zy))
    parts, i = [], 0
    while i < len(rows):
        k = rng.randint(1, 900)
        parts.append(rows[i:i + k])
        i += k
    parts.insert(2, [])   # a partition without rows
    (row,) = _final(_all_fns_plan(), parts, _exact_bufs)
    _check(row, rows)


def test_two_rank_partial_merge_equals_one_rank():
    api, desc = capi.product_api(), _all_fns_plan(keyed=True)
    rng = random.Random(9)
    rows = []
    for _ in range(3000):
        z = rng.gauss(0, 2)
        rows.append((bytes([97 + rng.randint(0, 3)]), (1e9 + z, 1e9 - 0.5 * z + rng.gauss(0, 1))))
    by = lambda sub: {k: [p for kk, p in sub if kk == k] for k in sorted({k for k, _ in sub})}

    def partial(sub):
        g = by(sub)
        return _partials(desc, [_exact_bufs(v) for v in g.values()], keys=list(g))
    one = capi.final_merge(api, desc, partial(rows))
    two = capi.final_merge(api, desc, capi.partial_merge_raw(api, desc, partial(rows[:1700]) + partial(rows[1700:])))
    assert sorted(r[0] for r in one) == sorted(r[0] for r in two)
    for a, b in zip(sorted(one), sorted(two)):
        g = by(rows)[a[0]]
        scale = R.exact_scale(g)
        for fn, x, y in zip(FNS, a[1:], b[1:]):
            assert R.close(fn, y, x, scale), (fn, x, y)
        _check(a[1:], g)


def test_naive_raw_sums_miss_the_bar():
    rng = random.Random(4)
    rows = []
    for _ in range(10000):
        z = rng.gauss(0, 1)
        rows.append((1e9 + z, 1e9 + 0.9 * z + math.sqrt(1 - 0.81) * rng.gauss(0, 1)))
    scale = R.exact_scale(rows)
    for fn in FNS:
        assert not R.close(fn, R.naive(fn, rows), R.exact(fn, rows), scale), fn


def _refused(build_plan):
    b = PlanBuilder()
    x, y, i = b.col(T.DOUBLE, 0, True), b.col(T.DOUBLE, 1, True), b.col(T.INT, 2, False)
    build_plan(b, x, y, i)
    rc, msg, _ = _codegen(b.build())
    return rc, msg


@pytest.mark.parametrize("case", ["not_pair", "pair_in_filter", "pair_as_key", "pair_projected", "pair_under_cast",
                                  "pair_under_add", "pair_under_isnull", "pair_in_sum", "pair_in_stddev", "pair_in_count",
                                  "int_child", "float_child", "pair_not_double", "update_set"])
def test_pair_misuse_is_refused(case):
    def plan(b, x, y, i):
        p = b.pair(x, y)
        if case == "not_pair":
            b.agg(AggFn.CORR, x)
        elif case == "pair_in_filter":
            b.filter(p.is_not_null()).count()
        elif case == "pair_as_key":
            b.group_by(p).count()
        elif case == "pair_projected":
            b.project(p)
        elif case == "pair_under_cast":
            b.sum(p.cast(T.LONG))
        elif case == "pair_under_add":
            b.sum(p + x)
        elif case == "pair_under_isnull":
            b.filter(p.is_null()).corr(x, y)
        elif case == "pair_in_sum":
            b.sum(p)
        elif case == "pair_in_stddev":
            b.stddev(p)
        elif case == "pair_in_count":
            b.count(p)
        elif case == "int_child":
            b.covar_pop(i, y)
        elif case == "float_child":
            b.corr(x, b.col(T.FLOAT, 3, False))
        elif case == "pair_not_double":
            b.agg(AggFn.COVAR_SAMP, E(b, Op.PAIR, T.LONG, x, y))
        else:
            b.update({0: p})
    rc, msg = _refused(plan)
    assert rc == capi.SD_ERR_INVALID, (case, rc, msg)


def test_cast_children_are_accepted():
    b = PlanBuilder()
    i, f = b.col(T.INT, 0, True), b.col(T.FLOAT, 1, False)
    b.covar_pop(i.cast(T.DOUBLE), f.cast(T.DOUBLE)).corr(i.cast(T.DOUBLE), f.cast(T.DOUBLE))
    rc, src, _ = _codegen(b.build())
    assert rc == 0, src


def test_covariance_plans_share_shifts_and_sums():
    b = PlanBuilder()
    x, y = b.col(T.DOUBLE, 0, True), b.col(T.DOUBLE, 1, False)
    b.covar_pop(x, y).covar_samp(x, y).corr(x, y).count()
    rc, src, _ = _codegen(b.build())
    assert rc == 0, src
    assert "NSHIFT = 2;" in src and "NPAIR = 1;" in src
    assert src.count("sd::shift_cand") == 2
    # n, S_x, S_y, S_xy, S_xx, S_yy, and the COUNT(*) slot
    assert "NSLOT = 7;" in src
    # a STDDEV of x keeps its own x-gated sums and shift; a second pair (y, x) its own
    b = PlanBuilder()
    x, y = b.col(T.DOUBLE, 0, True), b.col(T.DOUBLE, 1, False)
    b.corr(x, y).stddev(x).covar_pop(y, x)
    rc, src, _ = _codegen(b.build())
    assert rc == 0, src
    assert "NSHIFT = 5;" in src and "NPAIR = 2;" in src
    assert src.count("sd::shift_cand") == 5


def _plans_for_nvrtc():
    out = []
    for keyed in ("none", "dense", "hash"):
        b = PlanBuilder()
        x, q, y = b.col(T.DOUBLE, 0, True), b.col(T.INT, 2, False), b.col(T.DOUBLE, 3, True)
        b.filter(q > b.lit(T.INT))
        if keyed == "dense":
            b.group_by(b.col(T.STRING, 1, True))
        elif keyed == "hash":
            b.group_by(q)
        b.covar_pop(x, y).covar_samp(x, y).corr(x, q.cast(T.DOUBLE)).stddev(x).sum(x).count()
        out.append(b.build())
    return out


def test_covariance_plans_compile_with_nvrtc():
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
    rows = [(1.0, 2.0), (2.0, 4.0), (4.0, 5.0)]
    n, mx, my, ck, xmk, ymk = R.exact_buffers(rows)
    assert (n, mx, my) == (3, R.Fraction(7, 3), R.Fraction(11, 3))
    assert ck == sum((R.Fraction(x) - mx) * (R.Fraction(y) - my) for x, y in rows)
