"""DECIMAL columns wider than 18 digits on the device: records [int32 len][BigInteger.toByteArray()] (enc/Uncompressed.scala:
330-345) scanned, compared, grouped and aggregated, checked against exact Python integer arithmetic on the same values."""
import numpy as np
import pytest

from snappydata_b200 import capi
from snappydata_b200.column_format import (ColumnBatch, SqlType as T, compress_lz4, encode_column, encode_wide_decimal,
                                           stats_row, column_stats, wide_decimal_stats)
from snappydata_b200.plan import PlanBuilder

pytestmark = pytest.mark.gpu

P, S = 38, 18
EDGES = [0, -1, 127, 128, -129, 10 ** 38 - 1, -(10 ** 38 - 1)]


@pytest.fixture(scope="module")
def api():
    a = capi.product_api()
    a.check(a.init(0))
    return a


def values(n, seed, nullable, all_null_tile=False, max_digits=36):
    r = np.random.default_rng(seed)
    digits = r.integers(0, max_digits + 1, n)
    vals = [int(r.integers(0, 10 ** min(int(d), 18) + 1)) * 10 ** max(0, int(d) - 18) * (1 if r.random() < 0.6 else -1) for d in digits]
    for i, e in enumerate(EDGES[: min(n, len(EDGES))]):
        vals[i] = e if max_digits >= 38 else vals[i]
    nulls = (r.random(n) < 0.2) if nullable else None
    if nullable and all_null_tile and n > 2048:
        nulls[1024:2048] = True
    return vals, nulls


def batch(vals, nulls, keys, lz4=False, batch_id=0):
    n = len(vals)
    col = encode_wide_decimal(vals, nulls)
    if lz4:
        col = compress_lz4(col, force=True)
    kcol = encode_column(np.array(keys, dtype=object), T.STRING)
    st = stats_row(n, [wide_decimal_stats(vals, P, S, nulls), column_stats(np.array(keys, dtype=object), T.STRING)])
    return ColumnBatch(num_rows=n, columns=[col, kcol], stats=st, batch_id=batch_id)


def half_up_div(num, den):
    q, r = divmod(abs(num), den)
    if 2 * r >= den:
        q += 1
    return q if num >= 0 else -q


def expected_aggs(vals, nulls, p=P, s=S):
    live = [v for i, v in enumerate(vals) if nulls is None or not nulls[i]]
    if not live:
        return [None, None, None, 0, None]
    tot = sum(live)
    sum_v = None if abs(tot) >= 10 ** min(38, p + 10) else tot
    sp, ss = min(38, p + 4), min(38, s + 4)
    avg = half_up_div(tot * 10 ** (ss - s), len(live)) if sum_v is not None else None
    if avg is not None and abs(avg) >= 10 ** sp:
        avg = None
    return [sum_v, min(live), max(live), len(live), avg]


def agg_plan(nullable, filt=None):
    b = PlanBuilder()
    d = b.col(T.DECIMAL, 0, nullable, scale=S, precision=P)
    if filt is not None:
        b.filter(filt(b, d))
    b.sum(d).min(d).max(d).count(d).avg(d)
    return b.build()


def run(api, desc, batches, lits=(), store=False, nullable=True):
    pl = capi.Plan(api, desc).set_literals(list(lits))
    st = None
    if store:
        st = capi.Store(api, [(T.DECIMAL, nullable, P, S), (T.STRING, False)])
        for bt in batches:
            st.put(bt)
        pl.scan_store(st)
    else:
        for bt in batches:
            pl.submit(bt)
    raw = pl.finish_raw()
    out = pl.final_merge(raw)
    log = pl.launch_log()
    m = pl.metrics()
    pl.close()
    if st is not None:
        st.close()
    return out, log, m


@pytest.mark.parametrize("n", [1, 1023, 1025, 50_001, 200_000])
@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("store", [False, True])
def test_aggregates_exact(api, n, nullable, store):
    vals, nulls = values(n, n + 7 * nullable, nullable, all_null_tile=True, max_digits=30)
    bts = [batch(vals, nulls, [b"k"] * n, lz4=(n % 2 == 1))]
    out, log, _ = run(api, agg_plan(nullable), bts, store=store, nullable=nullable)
    assert out == [expected_aggs(vals, nulls)]
    paths = {k: sum(l["paths"][k] for l in log) for k in log[0]["paths"]}
    assert paths["fast_nulls" if nullable and nulls.any() else "all_fast"] >= 1, paths


def test_edge_values_min_max_and_overflow(api):
    vals = list(EDGES) + [5]
    out, _, _ = run(api, agg_plan(False), [batch(vals, None, [b"k"] * len(vals))], nullable=False)
    tot = sum(vals)
    assert out[0][1] == -(10 ** 38 - 1) and out[0][2] == 10 ** 38 - 1
    assert out[0][0] == tot   # the +-(10^38-1) pair cancels
    vals = [10 ** 38 - 1, 10 ** 38 - 1, 3]
    out, _, _ = run(api, agg_plan(False), [batch(vals, None, [b"k"] * 3)], nullable=False)
    assert out[0][0] is None and out[0][3] == 3 and out[0][4] is None   # |total| >= 10^38: NULL sum and average


def test_filters_comparisons_in_and_null_literals(api):
    n = 5000
    vals, nulls = values(n, 3, True, max_digits=38)
    lo, hi = vals[100], vals[200]
    lo, hi = min(lo, hi), max(lo, hi)
    bts = [batch(vals, nulls, [b"k"] * n)]
    desc = agg_plan(True, lambda b, d: (d >= b.lit(T.DECIMAL, P, S)) & (d < b.lit(T.DECIMAL, P, S)))
    out, _, _ = run(api, desc, bts, lits=[lo, hi])
    keep = [None if (nulls[i] or not (lo <= v < hi)) else v for i, v in enumerate(vals)]
    assert out == [expected_aggs([v or 0 for v in keep], np.array([v is None for v in keep]))]
    out, _, _ = run(api, desc, bts, lits=[None, hi])   # NULL literal: no row qualifies
    assert out == [[None, None, None, 0, None]]
    desc = agg_plan(True, lambda b, d: d.isin(3))
    picks = [vals[5], vals[9], vals[11]]
    out, _, _ = run(api, desc, bts, lits=picks)
    keep = [not nulls[i] and v in picks for i, v in enumerate(vals)]
    assert out == [expected_aggs(vals, np.array([not k for k in keep]))]
    out, _, _ = run(api, desc, bts, lits=[picks[0], None, picks[2]])
    keep = [not nulls[i] and v in (picks[0], picks[2]) for i, v in enumerate(vals)]
    assert out == [expected_aggs(vals, np.array([not k for k in keep]))]


def test_narrow_literal_cast_up(api):
    vals = [10 ** 20, 5 * 10 ** 18, -(10 ** 18), 3 * 10 ** 18]   # DECIMAL(38,18): 100.0, 5.0, -1.0, 3.0
    b = PlanBuilder()
    d = b.col(T.DECIMAL, 0, False, scale=S, precision=P)
    b.filter(d > b.lit(T.DECIMAL, 10, 2).cast(T.DECIMAL, P, S))
    b.sum(d).min(d).max(d).count(d).avg(d)
    out, _, _ = run(api, b.build(), [batch(vals, None, [b"k"] * 4)], lits=[400], nullable=False)   # 4.00
    assert out == [expected_aggs([10 ** 20, 5 * 10 ** 18], None)]


def test_reference_closed_form_decimal_28_25(api):
    """SHAByteBufferTest 'Big Decimal with precision > 18 as aggregate column': DECIMAL(28,25) of BigDecimal("" + .3*i)."""
    from decimal import Decimal
    strs = [repr(0.3 * i) for i in range(10)]
    vals = [int(Decimal(x).scaleb(25)) for x in strs]
    keys = [b"col%d" % (i // 5) for i in range(10)]
    col = encode_wide_decimal(vals)
    bt = ColumnBatch(num_rows=10, columns=[col, encode_column(np.array(keys, dtype=object), T.STRING)])
    b = PlanBuilder()
    d, k = b.col(T.DECIMAL, 0, False, scale=25, precision=28), b.col(T.STRING, 1, False)
    b.group_by(k)
    b.sum(d).avg(d)
    desc = b.build()
    assert desc.final_schema()[1:] == [(T.DECIMAL, 38, 25), (T.DECIMAL, 32, 29)]
    pl = capi.Plan(api, desc).set_literals([])
    pl.submit(bt)
    got = sorted(pl.final_merge(pl.finish_raw()))
    pl.close()
    sums = [sum(vals[:5]), sum(vals[5:])]
    # 3.0 and 10.5 up to the doubles' representation error (the reference checks them to 0.1; here the sums are exact)
    assert abs(sums[0] - 3 * 10 ** 25) < 10 ** 12 and abs(sums[1] - 105 * 10 ** 24) < 10 ** 12
    assert got == [[b"col0", sums[0], half_up_div(sums[0] * 10 ** 4, 5)], [b"col1", sums[1], half_up_div(sums[1] * 10 ** 4, 5)]]


def test_snap_3132_group_by_string_and_decimal_35_5(api):
    from decimal import ROUND_HALF_UP, Decimal
    n = 500
    c3 = [int(Decimal(17456567.576 * i).quantize(Decimal("0.00001"), rounding=ROUND_HALF_UP).scaleb(5)) for i in range(n)]
    name = [str(i % 10).encode() for i in range(n)]
    c2 = [i % 10 for i in range(n)]
    col3 = encode_wide_decimal(c3)
    bt = ColumnBatch(num_rows=n, columns=[encode_column(np.array(c2, dtype=np.int32), T.INT), col3,
                                          encode_column(np.array(name, dtype=object), T.STRING)])
    b = PlanBuilder()
    v2, v3, nm = b.col(T.INT, 0, False), b.col(T.DECIMAL, 1, False, scale=5, precision=35), b.col(T.STRING, 2, False)
    b.group_by(nm, v3)
    b.sum(v2)
    pl = capi.Plan(api, b.build()).set_literals([])
    pl.submit(bt)
    got = sorted(pl.final_merge(pl.finish_raw()))
    pl.close()
    want = {}
    for i in range(n):
        want[(name[i], c3[i])] = want.get((name[i], c3[i]), 0) + c2[i]
    assert got == sorted([list(k) + [v] for k, v in want.items()])


def test_hash_group_by_wide_and_string_over_wrapping_ring(api):
    n, nb = 1_000_000, 6
    r = np.random.default_rng(11)
    bts, allv, alln, allk = [], [], [], []
    for bi in range(nb):
        vals = [int(x) * 10 ** 20 + 7 for x in r.integers(-40, 40, n)]
        nulls = r.random(n) < 0.1
        keys = [b"g%d" % x for x in r.integers(0, 5, n)]
        bts.append(batch(vals, nulls, keys, batch_id=bi))
        allv += vals; alln += list(nulls); allk += keys
    b = PlanBuilder()
    d, k = b.col(T.DECIMAL, 0, True, scale=S, precision=P), b.col(T.STRING, 1, False)
    b.group_by(d, k)
    b.count().sum(d).min(d).max(d)
    for store in (False, True):
        out, log, _ = run(api, b.build(), bts, store=store)
        assert {l["accumulator"] for l in log} == {"hash"}
        want = {}
        for v, isn, kk in zip(allv, alln, allk):
            g = want.setdefault((None if isn else v, kk), [0, []])
            g[0] += 1
            if not isn:
                g[1].append(v)
        exp = sorted(([kv, kk, c, sum(l) if l else None, min(l) if l else None, max(l) if l else None]
                      for (kv, kk), (c, l) in want.items()), key=repr)
        assert sorted(out, key=repr) == exp


def test_projection_round_trip_decimal_35_15(api):
    for nullable in (False, True):
        vals, nulls = values(3000, 5, nullable, max_digits=35)
        b = PlanBuilder()
        d, k = b.col(T.DECIMAL, 0, nullable, scale=15, precision=35), b.col(T.STRING, 1, False)
        b.project(d, k)
        pl = capi.Plan(api, b.build()).set_literals([])
        pl.submit(batch(vals, nulls, [b"x"] * len(vals)))
        got = pl.finish()
        pl.close()
        want = [None if (nulls is not None and nulls[i]) else v for i, v in enumerate(vals)]   # rows come in no fixed order
        assert sorted((r[0] for r in got), key=repr) == sorted(want, key=repr) and all(r[1] == b"x" for r in got)


def test_stats_skipping_on_wide_bounds(api):
    bts = []
    for bi in range(4):
        vals = [(bi * 1000 + j) * 10 ** 20 for j in range(1000)]
        bts.append(batch(vals, None, [b"k"] * 1000, batch_id=bi))
    desc = agg_plan(False, lambda b, d: d >= b.lit(T.DECIMAL, P, S))
    lit = 2500 * 10 ** 20
    out, _, m = run(api, desc, bts, lits=[lit], nullable=False)
    live = [(bi * 1000 + j) * 10 ** 20 for bi in range(4) for j in range(1000) if (bi * 1000 + j) * 10 ** 20 >= lit]
    assert out == [expected_aggs(live, None)]
    assert m["columnBatchesSkipped"] == 2


def test_store_refusals_and_delete(api):
    vals, nulls = values(4000, 9, True, max_digits=38)
    st = capi.Store(api, [(T.DECIMAL, True, P, S), (T.STRING, False)])
    st.put(batch(vals, nulls, [b"k"] * 4000))
    with pytest.raises(capi.SdError) as ei:
        st.encode_batch(10, {0: (np.zeros(10, dtype=np.int64), None)})
    assert ei.value.code == 2
    assert st.num_batches() == 1
    b = PlanBuilder()   # DELETE WHERE d < 0, then scan: the remaining rows are the non-negative ones
    d = b.col(T.DECIMAL, 0, True, scale=S, precision=P)
    b.filter(d < b.lit(T.DECIMAL, P, S))
    dp = capi.Plan(api, b.delete().build())
    deleted = dp.delete_store(st, [0])
    dp.close()
    live = [None if (nulls[i] or v < 0) else v for i, v in enumerate(vals)]
    assert deleted == sum(1 for i, v in enumerate(vals) if not nulls[i] and v < 0)
    for reclaim in (False, True):
        if reclaim:
            st.reclaim(1.0)
        pl = capi.Plan(api, agg_plan(True)).set_literals([])
        pl.scan_store(st)
        out = pl.final_merge(pl.finish_raw())
        pl.close()
        keep = [i for i, v in enumerate(vals) if not (not nulls[i] and v < 0)]
        assert out == [expected_aggs([vals[i] for i in keep], np.array([bool(nulls[i]) for i in keep]))]
    with pytest.raises(capi.SdError) as ei:
        st.compact(0.0)
    assert ei.value.code == 2
    st.close()


@pytest.mark.parametrize("n", [1025, 50_001])
@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("lz4", [False, True])
def test_record_lengths_1_to_16(api, n, nullable, lz4):
    r = np.random.default_rng(n + nullable + 2 * lz4)
    vals = list(EDGES)
    while len(vals) < n:   # a magnitude of every record length 1..16, both signs
        ln = int(r.integers(1, 17))
        v = int(r.integers(0, 2 ** 62)) << max(0, 8 * ln - 64)
        vals.append(v % min(2 ** (8 * ln - 1), 10 ** 38) * (1 if r.random() < 0.5 else -1))
    vals = vals[:n]
    nulls = (r.random(n) < 0.2) if nullable else None
    for store in (False, True):
        out, _, _ = run(api, agg_plan(nullable), [batch(vals, nulls, [b"k"] * n, lz4=lz4)], store=store, nullable=nullable)
        assert out == [expected_aggs(vals, nulls)]


def test_plan_and_store_must_agree_on_the_decimal_layout(api):
    vals = [1, -2, 10 ** 30]
    wide_store = capi.Store(api, [(T.DECIMAL, False, P, S), (T.STRING, False)])
    wide_store.put(batch(vals, None, [b"k"] * 3))
    narrow_store = capi.Store(api, [(T.DECIMAL, False), (T.STRING, False)])   # precision 18
    from snappydata_b200.column_format import encode_uncompressed
    narrow_store.put(ColumnBatch(num_rows=3, columns=[encode_uncompressed(np.array([1, -2, 3], dtype=np.int64), T.DECIMAL),
                                                      encode_column(np.array([b"k"] * 3, dtype=object), T.STRING)]))
    b = PlanBuilder()
    nd = b.col(T.DECIMAL, 0, False, scale=S, precision=18)
    b.sum(nd)
    narrow_plan = b.build()
    b = PlanBuilder()
    wd = b.col(T.DECIMAL, 0, False, scale=4, precision=P)
    b.sum(wd)
    other_scale = b.build()
    for desc, st in ((agg_plan(False), narrow_store), (narrow_plan, wide_store), (other_scale, wide_store)):
        pl = capi.Plan(api, desc).set_literals([])
        with pytest.raises(capi.SdError) as ei:
            pl.scan_store(st)
        assert ei.value.code == 1
        assert pl.launch_log() == []
        pl.close()
    b = PlanBuilder()   # the UPDATE / DELETE scan checks it too
    d = b.col(T.DECIMAL, 0, False, scale=S, precision=P)
    b.filter(d.is_not_null())
    dp = capi.Plan(api, b.delete().build())
    with pytest.raises(capi.SdError) as ei:
        dp.delete_store(narrow_store, [])
    assert ei.value.code == 1
    dp.close()
    out, _, _ = run(api, agg_plan(False), [batch(vals, None, [b"k"] * 3)], nullable=False)
    assert out == [expected_aggs(vals, None)]
    wide_store.close()
    narrow_store.close()


def test_refusals_leave_the_store_unchanged(api):
    vals, nulls = values(3000, 21, True, max_digits=38)
    st = capi.Store(api, [(T.DECIMAL, True, P, S), (T.STRING, False)])
    st.put(batch(vals, nulls, [b"k"] * 3000))

    def state():
        pl = capi.Plan(api, agg_plan(True)).set_literals([])
        pl.scan_store(st)
        res = pl.final_merge(pl.finish_raw())
        pl.close()
        return st.num_batches(), st.get_stats(0), st.get_buffer(0, 0), res

    before = state()
    assert before[3] == [expected_aggs(vals, nulls)]
    with pytest.raises(capi.SdError) as ei:   # device ingest of a wide column
        st.encode_batch(10, {0: (np.zeros(10, dtype=np.int64), None)})
    assert ei.value.code == 2
    b = PlanBuilder()   # a DELETE makes the batch dirty; compaction would have to rewrite the wide column
    d = b.col(T.DECIMAL, 0, True, scale=S, precision=P)
    b.filter(d.is_null())
    dp = capi.Plan(api, b.delete().build())
    dp.delete_store(st, [])
    dp.close()
    after_delete = state()
    with pytest.raises(capi.SdError) as ei:
        st.compact(0.0)
    assert ei.value.code == 2 and "batch" in str(ei.value) and "column 0" in str(ei.value)
    assert state() == after_delete
    assert after_delete[3] == [expected_aggs([v for i, v in enumerate(vals) if not nulls[i]], None)]
    # an update delta on a wide column is kept but refused when a plan scans that column
    dst = capi.Store(api, [(T.DECIMAL, True, P, S), (T.STRING, False)])
    bt = batch(vals, nulls, [b"k"] * 3000)
    bt.delta0 = {0: b"\0" * 32}
    dst.put(bt)
    pl = capi.Plan(api, agg_plan(True)).set_literals([])
    with pytest.raises(capi.SdError) as ei:
        pl.scan_store(dst)
    assert ei.value.code == 2 and "column 0" in str(ei.value)
    pl.close()
    dst.close()
    st.close()
