"""Host-only checks of FIRST / LAST (with and without ignoreNulls): the two restatements of Spark's rule in
tests/first_last_reference.py against each other on every batch kind, the product's host merges against Spark's merge rule,
the partial-row schemas, the pair layout and sharing in the generated plan, the refusals, the generated source of plans
without these functions (unchanged), and NVRTC compiles of FIRST / LAST plans."""
import hashlib
import itertools
import struct

import pytest

import first_last_reference as R
import kernel_cases as kc
from snappydata_b200 import capi
from snappydata_b200.capi import AggFn
from snappydata_b200.column_format import SqlType as T, unsafe_row
from snappydata_b200.plan import PlanBuilder, q1_plan
from test_moment_aggregates import _codegen

TYPED = ["i", "l", "f", "d", "m", "s", "b", "t", "sh", "dt", "k"]
ALL_AGGS = [(AggFn.COUNT_STAR, None)] + [(fn, c) for c in TYPED for fn in R.ORDER_FNS]


def _batches(kinds, sizes, first_null=True):
    out = []
    for i, (kind, n) in enumerate(zip(kinds, sizes)):
        b, raw = kc.make_batch(n, kind, seed=4100 + i, groups=5, batch_id=i)
        if first_null and "d" in raw.nulls and raw.nulls["d"].any():   # NULL at the first and the last qualifying positions
            raw.nulls["d"][[0, n - 1]] = True
        out.append(raw)
    return out


@pytest.mark.parametrize("keys", [[], ["k"], ["h"]], ids=["nokey", "string_key", "int_key"])
@pytest.mark.parametrize("lit", [None, 600])
def test_row_rule_and_numpy_restatement_agree(keys, lit):
    """every mode, every type, every batch kind (NULLs, depth-0 / depth-1 deltas over boundary rows, delete masks)"""
    raws = _batches(kc.KINDS, [1, 2049, 3 * 2048 + 77, 1025, 513, 2047, 4096])
    a = R.update_rows(keys, ALL_AGGS, raws, lit)
    b = R.numpy_rows(keys, ALL_AGGS, raws, lit)
    R.assert_rows_equal(a, b, len(keys), f"keys={keys} lit={lit}")
    assert any(r[j] is None and r[j + 1] is True for r in a for j in range(len(keys) + 1, len(r) - 1)), "a winner with a NULL value"


def test_partial_and_final_schemas():
    d = R.desc(["k"], [(AggFn.FIRST, "d"), (AggFn.LAST_IGNORE_NULLS, "s"), (AggFn.FIRST, "m"), (AggFn.COUNT_STAR, None)])
    assert d.partial_schema() == [T.STRING, T.DOUBLE, T.BOOLEAN, T.STRING, T.BOOLEAN, (T.DECIMAL, 18, 2), T.BOOLEAN, T.LONG]
    assert d.final_schema() == [T.STRING, T.DOUBLE, T.STRING, (T.DECIMAL, 18, 2), T.LONG]


def _partials(desc, rows):
    schema = desc.partial_schema()
    out = b""
    for vals in rows:
        row = unsafe_row(list(zip(schema, vals)))
        out += struct.pack("<q", len(row)) + row
    return out


@pytest.mark.parametrize("fn", R.ORDER_FNS)
def test_host_merges_follow_sparks_merge_rule_in_every_order(fn):
    """partial rows of one group in every order, including partitions whose valueSet is false and NULL values that are set"""
    d = R.desc(["h"], [(fn, "d")])
    parts = [[7, None, False], [7, 1.5, True], [7, None, True], [7, -0.0, True], [7, None, False]]
    api = capi.product_api()
    for order in itertools.permutations(range(len(parts))):
        rows = [parts[i] for i in order]
        want = rows[0][1:]
        for r in rows[1:]:
            want = R.merge(fn, want, r[1:])
        (got,) = capi.final_merge(api, d, _partials(d, rows))
        assert R.canon(got[1]) == R.canon(want[0]), (order, got, want)
        merged = capi.parse_row_stream(capi.partial_merge_raw(api, d, _partials(d, rows)), d.partial_schema())
        assert [R.canon(x) for x in merged[0]] == [R.canon(x) for x in [7] + want], (order, merged, want)


def test_no_key_merge_of_no_partitions_is_null_and_not_set():
    d = R.desc([], [(AggFn.FIRST, "s"), (AggFn.LAST_IGNORE_NULLS, "d")])
    api = capi.product_api()
    assert capi.final_merge(api, d, b"") == [[None, None]]
    assert capi.parse_row_stream(capi.partial_merge_raw(api, d, b""), d.partial_schema()) == [[None, False, None, False]]


def test_pairs_are_even_shared_per_function_and_input():
    b = PlanBuilder()
    x, y, s = b.col(T.DOUBLE, 0, True), b.col(T.INT, 1, False), b.col(T.STRING, 2, True)
    b.group_by(b.col(T.LONG, 3, False))
    b.count().first(x).first(x).last(x).first(x, ignore_nulls=True).sum(y).first(s).last(s, ignore_nulls=True).first(x)
    rc, src, _ = _codegen(b.build())
    assert rc == 0, src
    assert "static constexpr int NORDER = 5;" in src   # FIRST(x) shared three times; LAST(x), FIRST(x) IGNORE NULLS apart
    ops = src.split("slot_op(int s) { return ")[1].split(";")[0]
    table = {int(a): int(o) for a, o in (t.split(" ? ") for t in ops.split(" : ")[:-1] for t in [t.replace("s == ", "")])}
    nslot = int(src.split("NSLOT = ")[1].split(";")[0])
    assert nslot % 2 == 0
    keys = [s for s, op in table.items() if op in (10, 11)]
    assert len(keys) == 5 and all(s % 2 == 0 and table.get(s + 1) == 12 for s in keys), table


def _refused(desc):
    rc, msg, _ = _codegen(desc)
    return rc, msg


def test_refusals_of_string_and_wide_decimal_expressions():
    b = PlanBuilder()
    b.col(T.INT, 0, False)
    b.first(b.lit(T.STRING))
    rc, msg = _refused(b.build())
    assert rc == 2 and "FIRST / LAST" in msg, msg
    b = PlanBuilder()
    m = b.col(T.DECIMAL, 0, True, scale=2, precision=12)
    b.last(m.cast(T.DECIMAL, 38, 2), ignore_nulls=True)
    rc, msg = _refused(b.build())
    assert rc == 2 and "FIRST / LAST" in msg, msg
    b = PlanBuilder()   # a wide DECIMAL column and a STRING column are fine
    b.first(b.col(T.DECIMAL, 0, True, scale=2, precision=38)).last(b.col(T.STRING, 1, True))
    assert _codegen(b.build())[0] == 0


def _hash_plan():
    b = PlanBuilder()
    k, d, v, s = b.col(T.INT, 0, True), b.col(T.DATE, 1, False), b.col(T.DOUBLE, 2, True), b.col(T.STRING, 3, True)
    b.filter((d >= b.lit(T.DATE)) & s.is_not_null())
    b.group_by(k, d)
    b.count().sum(v).avg(v).min(v).max(k).count(v).min(s)
    return b.build()


def _moment_plan():
    b = PlanBuilder()
    x, k = b.col(T.DOUBLE, 0, True), b.col(T.STRING, 1, False)
    b.group_by(k)
    b.stddev(x).kurtosis(x).var_pop(x.cast(T.DOUBLE)).count()
    return b.build()


def _covariance_plan():
    b = PlanBuilder()
    x, y, k = b.col(T.DOUBLE, 0, True), b.col(T.DOUBLE, 1, True), b.col(T.LONG, 2, False)
    b.group_by(k)
    b.covar_pop(x, y).corr(x, y).sum(x)
    return b.build()


# sha256 of the generated source of the parent commit (before FIRST / LAST existed)
UNCHANGED = {
    "q1": (q1_plan, "96cc39edb7d18a0108a3cd04d68cc2e2a90bbf51fee38c92a5e52132e8157ec5"),
    "hash": (_hash_plan, "52537eacd4d8f72286443a2f4fe8cc659ce8c3abda53f6dd09dd9b0879c581b1"),
    "moment": (_moment_plan, "7c71d82e3491f661a7b77c8fcde830a5edb66d4a4cbfb766f2dff2825a59f342"),
    "covariance": (_covariance_plan, "b4cfda742ee8057ee3e9d58e107a832fea908d32c5e05b55649b78a24190249d"),
}


@pytest.mark.parametrize("label", list(UNCHANGED))
def test_generated_source_of_plans_without_first_last_is_unchanged(label):
    make, sha = UNCHANGED[label]
    rc, src, _ = _codegen(make())
    assert rc == 0, src
    assert "NORDER" not in src
    assert hashlib.sha256(src.encode()).hexdigest() == sha, label


def _first_last_plans():
    out = {}
    b = PlanBuilder()   # no keys: every type, the register / shuffle / CTA / last-CTA combines
    cs = {n: b.col(kc.TYPE[n], kc.COL[n], kc.NULLABLE[n], scale=2 if kc.TYPE[n] == T.DECIMAL else 0) for n in TYPED}
    b.filter(cs["i"] > b.lit(T.INT))
    b.count()
    for n in TYPED:
        b.first(cs[n]).last(cs[n], ignore_nulls=True)
    out["nokey"] = b.build()
    b = PlanBuilder()   # dense table: private / shared-atomic / global-atomic pairs
    k, d, s = b.col(T.STRING, 0, True), b.col(T.DOUBLE, 1, True), b.col(T.STRING, 2, True)
    b.group_by(k)
    b.first(d).last(d).first(s, ignore_nulls=True).count()
    out["dense"] = b.build()
    b = PlanBuilder()   # hash table, wide DECIMAL by reference
    h, w, t = b.col(T.LONG, 0, False), b.col(T.DECIMAL, 1, True, scale=2, precision=38), b.col(T.TIMESTAMP, 2, True)
    b.group_by(h)
    b.first(w).last(w, ignore_nulls=True).first(t).last(t).sum(t)
    out["hash"] = b.build()
    return out


@pytest.mark.parametrize("label", ["nokey", "dense", "hash"])
def test_first_last_plans_compile_with_nvrtc(label):
    pytest.importorskip("cuda.bindings.nvrtc")
    from test_jit_compiles import _codegen as codegen_variant, _compile
    seen = set()
    for slow, litnull in ((0, 0), (1, 0), (0, 1), (1, 1)):
        source, _, name = codegen_variant(_first_last_plans()[label], slow, litnull)
        assert "NORDER" in source and name not in seen
        seen.add(name)
        _compile(source, name)
