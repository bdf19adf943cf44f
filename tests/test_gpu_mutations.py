"""UPDATE / DELETE over a resident store on the device (sd_plan_update_store / sd_plan_delete_store): the merged delta and
delete-mask bytes against the host fixture writer + sd_delta_merge, the rows changed against numpy, query results after each
statement against the CPU oracle over host ColumnBatches carrying the same bytes, the stats-row merge, whole-batch deletes,
atomicity against a concurrent query, and the error rules (a failing statement leaves the store as it was)."""
import ctypes as C
import struct
import threading

import numpy as np
import pytest

from snappydata_b200 import capi, lineitem, plan as P
from snappydata_b200.capi import SdError
from snappydata_b200.column_format import (ColumnBatch, SqlType as T, column_stats, encode_delete, encode_delta, parse_unsafe_row,
                                           stats_row)
from snappydata_b200.plan import L_DISCOUNT, L_QUANTITY, L_SHIPDATE, PlanBuilder

from helpers import assert_rowsets_match

pytestmark = pytest.mark.gpu

RPB = 20_000
NB = 20
SEED = 11


def _merge(api, t, new, existing, num_rows):
    f = api.lib.sd_delta_merge
    f.restype = C.c_int
    f.argtypes = [C.POINTER(capi.sd_column), C.c_char_p, C.c_int64, C.c_char_p, C.c_int64, C.c_int32, C.c_int32, C.c_char_p, C.c_int64,
                  C.POINTER(C.c_int64)]
    col = capi.sd_column(int(t), 0, 0, 0, 0)
    out, ln = C.create_string_buffer(len(new) + len(existing) + 64), C.c_int64()
    api.check(f(C.byref(col), new, len(new), existing, len(existing), 1, num_rows, out, len(out), C.byref(ln)))
    return out.raw[: ln.value]


class Model:
    """The table on the host: per batch the effective values, the live rows, and the delta / mask bytes it should hold."""

    def __init__(self, rng, api):
        # the base table generated on the device, pulled back once, decorated with deltas / deletes on the host and re-put
        # (the way workloads.run_c5 builds its table)
        gen = capi.Store(api, lineitem.LINEITEM_SCHEMA)
        gen.gen_lineitem(0, NB * RPB, RPB, 4, SEED, lineitem.Q1_COLUMN_MASK)
        self.batches = []
        for i in range(NB):
            nrows, bucket, bid = gen.batch_info(i)
            cols = [None] * 16
            for c in (L_QUANTITY, L_DISCOUNT, L_SHIPDATE, P.L_EXTENDEDPRICE, P.L_TAX, P.L_RETURNFLAG, P.L_LINESTATUS):
                cols[c] = gen.get_buffer(i, c)
            self.batches.append(ColumnBatch(num_rows=nrows, columns=cols, batch_id=bid, bucket_id=bucket))
        gen.close()
        self.vals, self.live, self.delta0, self.delta1, self.mask = [], [], [], [], []
        for i, b in enumerate(self.batches):
            v = lineitem.lineitem_values(i * RPB, RPB, SEED)
            eff = {L_QUANTITY: v["l_quantity"].copy(), L_DISCOUNT: v["l_discount"].copy(), L_SHIPDATE: v["l_shipdate"].copy(),
                   P.L_EXTENDEDPRICE: v["l_extendedprice"]}
            d0, d1 = {}, {}
            if i % 3 == 1:   # existing depth-1 then depth-0 deltas (depth 0 wins), like a table that took earlier updates
                for depth, store_d in ((1, d1), (0, d0)):
                    for c in (L_DISCOUNT, L_QUANTITY):
                        pos = np.sort(rng.choice(RPB, 700, replace=False)).astype(np.int32)
                        new = (rng.integers(0, 11, 700) / 100.0) if c == L_DISCOUNT else rng.integers(1, 51, 700).astype(np.float64)
                        store_d[c] = encode_delta(RPB, pos, new, T.DOUBLE)
                        eff[c][pos] = new
            b.delta0, b.delta1 = dict(d0), dict(d1)
            live = np.ones(RPB, bool)
            if i % 4 == 2:
                dp = np.sort(rng.choice(RPB, 500, replace=False)).astype(np.int32)
                b.delete_mask = encode_delete(RPB, dp)
                live[dp] = False
            self.mask.append(b.delete_mask)
            cs = [(T.LONG, None, None, 0)] * 16
            for c in (L_QUANTITY, L_DISCOUNT, P.L_EXTENDEDPRICE, P.L_TAX):
                cs[c] = column_stats(eff[c] if c in eff else v["l_tax"], T.DOUBLE)
            cs[L_SHIPDATE] = column_stats(v["l_shipdate"], T.DATE)
            for c in (P.L_RETURNFLAG, P.L_LINESTATUS, 11, 12, 13, 14, 15):
                cs[c] = (T.DATE if c in (11, 12) else T.STRING, None, None, 0)
            for c in (0, 1, 2):
                cs[c] = (T.LONG, None, None, 0)
            cs[3] = (T.INT, None, None, 0)
            b.stats = stats_row(RPB, cs, has_deltas=bool(d0 or d1))
            self.vals.append(eff)
            self.live.append(live)
            self.delta0.append(dict(d0))
            self.delta1.append(dict(d1))


@pytest.fixture()
def table(gpu_api):
    rng = np.random.default_rng(3)
    m = Model(rng, gpu_api)
    store = capi.Store(gpu_api, lineitem.LINEITEM_SCHEMA)
    for b in m.batches:
        store.put(b)
    yield m, store
    store.close()


def _update_plan(assign, where):
    """assign(b, cols) -> {table ordinal: expr}; where(b, cols) -> predicate or None."""
    b = PlanBuilder()
    cols = {c: b.col(lineitem.LINEITEM_SCHEMA[c][0], c) for c in (L_QUANTITY, L_DISCOUNT, L_SHIPDATE)}
    w = where(b, cols)
    if w is not None:
        b.filter(w)
    if assign is None:
        b.delete()
    else:
        b.update(assign(b, cols))
    return b.build()


def _host_batches(m, store):
    """ColumnBatches carrying the bytes the store now holds (for the oracle)."""
    out = []
    for i, b in enumerate(m.batches):
        d0 = {c: store.get_delta(i, c, 0) for c in (L_QUANTITY, L_DISCOUNT) if c in m.delta0[i]}
        d1 = {c: store.get_delta(i, c, 1) for c in (L_QUANTITY, L_DISCOUNT) if c in m.delta1[i]}
        out.append(ColumnBatch(num_rows=b.num_rows, columns=b.columns, stats=None, delta0=d0, delta1=d1,
                               delete_mask=m.mask[i], batch_id=b.batch_id, bucket_id=b.bucket_id))
    return out


def _check_queries(gpu_api, m, store, plans):
    from oracle import oracle
    hb = _host_batches(m, store)
    for (desc, lits, nkeys), gp in plans:
        got = capi.parse_row_stream(gp.execute_store_raw(store, gp.literal_array(lits), len(lits)), desc.partial_schema())
        op = oracle.plan(desc).set_literals(lits)
        for b in hb:
            if b.delete_mask is None or struct.unpack_from("<i", b.delete_mask, 8)[0] < b.num_rows:
                op.submit(b)
        assert_rowsets_match(got, op.finish(), nkeys)
        op.close()
    # Q6 against numpy over the effective values
    d0, d1, lo, hi, q = P.Q6_LITERALS
    want = 0.0
    for i in range(NB):
        v = m.vals[i]
        sel = m.live[i] & (v[L_SHIPDATE] >= d0) & (v[L_SHIPDATE] < d1) & (v[L_DISCOUNT] >= lo) & (v[L_DISCOUNT] <= hi) & (v[L_QUANTITY] < q)
        want += float(np.sum(v[P.L_EXTENDEDPRICE][sel] * v[L_DISCOUNT][sel]))
    gp = plans[0][1]
    (got,), = capi.parse_row_stream(gp.execute_store_raw(store, gp.literal_array(P.Q6_LITERALS), 5), plans[0][0][0].partial_schema())
    assert got == pytest.approx(want, rel=1e-6)


def _apply_update(api, m, store, rows, new_vals, where_mask_fn):
    """Host restatement of one UPDATE: expected rows, delta bytes per touched (batch, column)."""
    total = 0
    for i in range(NB):
        v = m.vals[i]
        sel = m.live[i] & where_mask_fn(v)
        pos = np.nonzero(sel)[0].astype(np.int32)
        total += pos.shape[0]
        if not pos.shape[0]:
            continue
        news = {c: f(v)[pos] for c, f in new_vals.items()}
        for c, nv in news.items():
            nd = encode_delta(RPB, pos, nv, T.DOUBLE)
            m.delta0[i][c] = _merge(api, T.DOUBLE, nd, m.delta0[i][c], RPB) if c in m.delta0[i] else nd
            v[c][pos] = nv
    assert rows == total
    for i in range(NB):
        for c, want in m.delta0[i].items():
            assert store.get_delta(i, c, 0) == want, (i, c)
        for c, want in m.delta1[i].items():
            assert store.get_delta(i, c, 1) == want, (i, c)


def test_update_delete_bytes_and_results(gpu_api):
    rng = np.random.default_rng(3)
    m = Model(rng, gpu_api)
    store = capi.Store(gpu_api, lineitem.LINEITEM_SCHEMA)
    for b in m.batches:
        store.put(b)
    plans = [((d, l, k), capi.Plan(gpu_api, d)) for d, l, k in ((P.q6_plan(), P.Q6_LITERALS, 0), (P.q1_plan(), P.Q1_LITERALS, 2))]
    _check_queries(gpu_api, m, store, plans)
    # UPDATE SET l_discount = l_discount + 0.01, l_quantity = 7 WHERE l_shipdate BETWEEN a AND b
    desc = _update_plan(lambda b, c: {L_DISCOUNT: c[L_DISCOUNT] + b.lit(T.DOUBLE), L_QUANTITY: b.lit(T.DOUBLE)},
                        lambda b, c: (c[L_SHIPDATE] >= b.lit(T.DATE)) & (c[L_SHIPDATE] <= b.lit(T.DATE)))
    assert desc.c.flags == capi.SD_PLAN_MUTATE and desc.targets == [L_DISCOUNT, L_QUANTITY]
    up = capi.Plan(gpu_api, desc)
    for a, bnd in ((8800, 9000), (8900, 9300)):   # the second statement overlaps the first
        rows = up.update_store(store, [a, bnd, 0.01, 7.0])
        _apply_update(gpu_api, m, store, rows, {L_DISCOUNT: lambda v: v[L_DISCOUNT] + 0.01, L_QUANTITY: lambda v: np.full(RPB, 7.0)},
                      lambda v: (v[L_SHIPDATE] >= a) & (v[L_SHIPDATE] <= bnd))
        _check_queries(gpu_api, m, store, plans)
    # DELETE WHERE l_quantity < k
    dp = capi.Plan(gpu_api, _update_plan(None, lambda b, c: c[L_QUANTITY] < b.lit(T.DOUBLE)))
    rows = dp.delete_store(store, [9.0])
    total = 0
    for i in range(NB):
        sel = m.live[i] & (m.vals[i][L_QUANTITY] < 9.0)
        total += int(sel.sum())
        if sel.any():
            m.live[i] &= ~sel
            m.mask[i] = encode_delete(RPB, np.nonzero(~m.live[i])[0])
        if m.mask[i] is not None:
            assert store.get_deletes(i) == m.mask[i], i
    assert rows == total
    _check_queries(gpu_api, m, store, plans)
    # stats of a touched batch: ColumnDelta.mergeStats restated
    st = parse_unsafe_row(store.get_stats(0), [T.INT] + [t for c in range(16) for t in (lineitem.LINEITEM_SCHEMA[c][0],) * 2 + (T.INT,)])
    assert st[0] < 0
    q = m.vals[0][L_QUANTITY]
    assert st[1 + 3 * L_QUANTITY] <= q[m.live[0]].min() and st[2 + 3 * L_QUANTITY] >= q[m.live[0]].max()
    for p in plans:
        p[1].close()
    up.close()
    dp.close()
    store.close()


def test_stats_widen_and_point_query_finds_new_value(gpu_api, table):
    m, store = table
    # a point query on l_quantity = 77 skips every batch before the update (bounds are 1..50)
    b = PlanBuilder()
    qc = b.col(T.DOUBLE, L_QUANTITY)
    b.filter(qc.eq(b.lit(T.DOUBLE)))
    b.count()
    pq = capi.Plan(gpu_api, b.build())
    cnt = lambda: capi.parse_row_stream(pq.execute_store_raw(store, pq.literal_array([77.0]), 1), pq.desc.partial_schema())[0][0]
    assert cnt() == 0
    assert pq.metrics()["columnBatchesSkipped"] == NB
    old_stats = [store.get_stats(i) for i in range(NB)]
    up = capi.Plan(gpu_api, _update_plan(lambda b, c: {L_QUANTITY: b.lit(T.DOUBLE)}, lambda b, c: c[L_SHIPDATE].eq(b.lit(T.DATE))))
    ship = 8100
    rows = up.update_store(store, [ship, 77.0])   # literal slots: the WHERE's first, then the SET values'
    want = sum(int((m.live[i] & (m.vals[i][L_SHIPDATE] == ship)).sum()) for i in range(NB))
    assert rows == want > 0
    assert cnt() == want
    touched = [i for i in range(NB) if (m.live[i] & (m.vals[i][L_SHIPDATE] == ship)).any()]
    assert pq.metrics()["columnBatchesSkipped"] == NB - len(touched)
    types = [T.INT] + [t for c in range(16) for t in (lineitem.LINEITEM_SCHEMA[c][0],) * 2 + (T.INT,)]
    for i in range(NB):
        old = parse_unsafe_row(old_stats[i], types)
        new = parse_unsafe_row(store.get_stats(i), types)
        if i not in touched:
            assert new == old
            continue
        n_new = int((m.live[i] & (m.vals[i][L_SHIPDATE] == ship)).sum())
        exp = list(old)
        exp[0] = -abs(old[0])
        f = 1 + 3 * L_QUANTITY
        exp[f] = min(old[f], 77.0)
        exp[f + 1] = max(old[f + 1], 77.0)
        nc = max(old[f + 2] - (n_new - 0), 0)
        exp[f + 2] = 1 if nc <= 0 and old[f + 2] > 0 else nc
        assert new == exp, i
    up.close()
    pq.close()


def test_whole_batch_delete(gpu_api, table):
    m, store = table
    q6 = capi.Plan(gpu_api, P.q6_plan())
    before = q6.execute_store_raw(store, q6.literal_array(P.Q6_LITERALS), 5)
    seen = q6.metrics()["columnBatchesSeen"]
    dp = capi.Plan(gpu_api, _update_plan(None, lambda b, c: None))
    rows = dp.delete_store(store, [], buckets=[0])   # every live row of the bucket-0 batches
    gone = [i for i in range(NB) if m.batches[i].bucket_id == 0]
    assert rows == sum(int(m.live[i].sum()) for i in gone)
    after = q6.execute_store_raw(store, q6.literal_array(P.Q6_LITERALS), 5)
    assert q6.metrics()["columnBatchesSeen"] == seen - len(gone)
    d0, d1, lo, hi, q = P.Q6_LITERALS
    want = 0.0
    for i in range(NB):
        if i in gone:
            continue
        v = m.vals[i]
        sel = m.live[i] & (v[L_SHIPDATE] >= d0) & (v[L_SHIPDATE] < d1) & (v[L_DISCOUNT] >= lo) & (v[L_DISCOUNT] <= hi) & (v[L_QUANTITY] < q)
        want += float(np.sum(v[P.L_EXTENDEDPRICE][sel] * v[L_DISCOUNT][sel]))
    (got,), = capi.parse_row_stream(after, q6.desc.partial_schema())
    assert got == pytest.approx(want, rel=1e-6) and before != after
    for i in gone:
        assert struct.unpack_from("<iii", store.get_deletes(i), 0) == (0, RPB, RPB)
    q6.close()
    dp.close()


def test_errors_leave_the_store_unchanged(gpu_api, table):
    m, store = table
    q6 = capi.Plan(gpu_api, P.q6_plan())
    snap = lambda: ([store.get_delta(i, c, 0) for i in range(NB) for c in m.delta0[i]], [store.get_stats(i) for i in range(NB)],
                    q6.execute_store_raw(store, q6.literal_array(P.Q6_LITERALS), 5))
    before = snap()
    where = lambda b, c: c[L_SHIPDATE] >= b.lit(T.DATE)

    def fails(code, fn):
        with pytest.raises(SdError) as e:
            fn()
        assert e.value.code == code
        assert snap() == before

    b = PlanBuilder()   # STRING target
    s = b.col(T.STRING, P.L_RETURNFLAG)
    b.filter(b.col(T.DATE, L_SHIPDATE) >= b.lit(T.DATE))
    b.update({P.L_RETURNFLAG: s})
    p1 = capi.Plan(gpu_api, b.build())
    fails(capi.SD_ERR_UNSUPPORTED, lambda: p1.update_store(store, [8000]))
    # NULL into the NOT NULL l_quantity
    p2 = capi.Plan(gpu_api, _update_plan(lambda b, c: {L_QUANTITY: b.lit(T.DOUBLE)}, where))
    fails(capi.SD_ERR_INVALID, lambda: p2.update_store(store, [8000, None]))
    # type mismatch: a DATE value into a DOUBLE column
    p3 = capi.Plan(gpu_api, _update_plan(lambda b, c: {L_QUANTITY: c[L_SHIPDATE]}, where))
    fails(capi.SD_ERR_INVALID, lambda: p3.update_store(store, [8000]))
    # a target that is not resident (l_orderkey was never put)
    p4 = capi.Plan(gpu_api, _update_plan(lambda b, c: {0: b.lit(T.LONG)}, where))
    fails(capi.SD_ERR_INVALID, lambda: p4.update_store(store, [8000, 5]))
    # wrong plan kinds
    fails(capi.SD_ERR_STATE, lambda: q6.update_store(store, P.Q6_LITERALS))
    fails(capi.SD_ERR_STATE, lambda: p2.scan_store(store))
    for p in (p1, p2, p3, p4, q6):
        p.close()


def test_atomicity_against_a_running_query(gpu_api, table):
    m, store = table
    b = PlanBuilder()
    b.sum(b.col(T.DOUBLE, L_QUANTITY))
    qdesc = b.build()
    nrows = sum(int(l.sum()) for l in m.live)
    base = sum(float(m.vals[i][L_QUANTITY][m.live[i]].sum()) for i in range(NB))
    up = capi.Plan(gpu_api, _update_plan(lambda b, c: {L_QUANTITY: c[L_QUANTITY] + b.lit(T.DOUBLE)}, lambda b, c: None))
    seen, stop, errors = [], threading.Event(), []

    def reader():
        try:
            gpu_api.check(gpu_api.init(0))
            qp = capi.Plan(gpu_api, qdesc)
            while not stop.is_set():
                (v,), = capi.parse_row_stream(qp.execute_store_raw(store, qp.literal_array([]), 0), qdesc.partial_schema())
                seen.append(v)
            qp.close()
        except Exception as e:   # reported below
            errors.append(e)

    t = threading.Thread(target=reader)
    t.start()
    for _ in range(6):
        assert up.update_store(store, [1.0]) == nrows
    stop.set()
    t.join()
    assert not errors, errors
    assert seen
    for v in seen:
        k = (v - base) / nrows
        assert abs(k - round(k)) < 1e-9 and 0 <= round(k) <= 6, v
    up.close()
