"""UPDATE / DELETE statements beyond the lineitem DOUBLE columns: the reference's closed forms for updates and deletes
(testDeltaStats, testBasicDeleteIter; the answers of tests/known_answer_cases.py) run as statements, nullable targets of the
narrow types with NULLs in the new values and in an existing Uncompressed / Dictionary depth-0 delta (bytes against
sd_delta_merge over two statements), batches appended while statements run, and a 1 % UPDATE / DELETE over a 60 M-row
store whose scan wraps the staged ring (every batch's bytes against the host construction)."""
import ctypes as C
import struct
import threading

import numpy as np
import pytest

from snappydata_b200 import capi, lineitem, plan as P
from snappydata_b200.capi import SdError
from snappydata_b200.column_format import (ColumnBatch, SqlType as T, column_stats, encode_delete, encode_delta, encode_uncompressed,
                                           parse_unsafe_row, stats_row)
from snappydata_b200.plan import L_DISCOUNT, L_QUANTITY, L_SHIPDATE, PlanBuilder

from known_answer_cases import _point_query

pytestmark = pytest.mark.gpu


def _run(p, lits, store):
    return capi.parse_row_stream(p.execute_store_raw(store, p.literal_array(lits), len(lits)), p.desc.partial_schema())


def _merge(api, t, nullable, new, existing, num_rows):
    f = api.lib.sd_delta_merge
    f.restype = C.c_int
    f.argtypes = [C.POINTER(capi.sd_column), C.c_char_p, C.c_int64, C.c_char_p, C.c_int64, C.c_int32, C.c_int32, C.c_char_p, C.c_int64,
                  C.POINTER(C.c_int64)]
    col = capi.sd_column(int(t), int(nullable), 0, 0, 0)
    out, ln = C.create_string_buffer(len(new) + len(existing) + 64), C.c_int64()
    api.check(f(C.byref(col), new, len(new), existing, len(existing), 1, num_rows, out, len(out), C.byref(ln)))
    return out.raw[: ln.value]


def test_delta_stats_closed_form_as_statements(gpu_api):
    """testDeltaStats: (10,100),(20,200); update col1 = 100 where col2 = 100; update col1 = 200 where col1 = 20;
    update col1 = col1 * 10.  Point queries go through stats skipping, so the merged stats row must admit the new values."""
    col1, col2 = np.array([10, 20], dtype=np.int64), np.array([100, 200], dtype=np.int64)
    store = capi.Store(gpu_api, [(T.LONG, False), (T.LONG, False)])
    store.put(ColumnBatch(num_rows=2, columns=[encode_uncompressed(col1, T.LONG), encode_uncompressed(col2, T.LONG)],
                          stats=stats_row(2, [column_stats(col1, T.LONG), column_stats(col2, T.LONG)])))
    q1, q2 = capi.Plan(gpu_api, _point_query(0, 1)), capi.Plan(gpu_api, _point_query(1, 0))

    def upd(where_col, expr):
        b = PlanBuilder()
        c = [b.col(T.LONG, 0), b.col(T.LONG, 1)]
        if where_col is not None:
            b.filter(c[where_col].eq(b.lit(T.LONG)))
        b.update({0: expr(b, c)})
        return capi.Plan(gpu_api, b.build())

    assert upd(1, lambda b, c: b.lit(T.LONG)).update_store(store, [100, 100]) == 1
    assert _run(q1, [100], store) == [[1, 100, 100]] and _run(q2, [100], store) == [[1, 100, 100]]
    assert _run(q1, [10], store)[0][0] == 0
    assert upd(0, lambda b, c: b.lit(T.LONG)).update_store(store, [20, 200]) == 1
    assert _run(q1, [200], store) == [[1, 200, 200]] and _run(q2, [200], store) == [[1, 200, 200]]
    assert store.get_delta(0, 0, 0) == encode_delta(2, [0, 1], np.array([100, 200], dtype=np.int64), T.LONG)
    assert upd(None, lambda b, c: c[0] * b.lit(T.LONG)).update_store(store, [10]) == 2
    assert _run(q1, [1000], store) == [[1, 1000, 100]] and _run(q1, [2000], store) == [[1, 2000, 200]]
    assert _run(q1, [100], store)[0][0] == 0 and _run(q2, [100], store) == [[1, 1000, 100]]
    st = parse_unsafe_row(store.get_stats(0), [T.INT, T.LONG, T.LONG, T.INT, T.LONG, T.LONG, T.INT])
    assert st == [-2, 10, 2000, 0, 100, 200, 0]
    store.close()


def test_basic_delete_iter_closed_form_as_statements(gpu_api):
    """testBasicDeleteIter: 50,000 rows (id, status, id % 10); delete where id % 10 = 0; two passes of
    `update id = id + 25000 where id <> 73`.  A BOOLEAN SET target is refused and leaves the store as it was."""
    n, per = 50_000, 10_000
    store = capi.Store(gpu_api, [(T.INT, False), (T.BOOLEAN, False), (T.INT, False)])
    for bid in range(n // per):
        ids = np.arange(bid * per, (bid + 1) * per, dtype=np.int32)
        store.put(ColumnBatch(num_rows=per, columns=[encode_uncompressed(ids, T.INT), encode_uncompressed((ids % 2) == 0, T.BOOLEAN),
                                                     encode_uncompressed(ids % 10, T.INT)], batch_id=bid))
    b = PlanBuilder()
    b.filter(b.col(T.INT, 2).eq(b.lit(T.INT)))
    b.delete()
    assert capi.Plan(gpu_api, b.build()).delete_store(store, [0]) == n // 10
    b = PlanBuilder()
    idc = b.col(T.INT, 0)
    b.filter(idc.ne(b.lit(T.INT)))
    b.update({0: idc + b.lit(T.INT)})
    up = capi.Plan(gpu_api, b.build())
    survivors = np.array([x for x in range(n) if x % 10 != 0], dtype=np.int64)
    for _ in range(2):
        assert up.update_store(store, [73, n // 2]) == len(survivors) - 1
    b = PlanBuilder()
    idc = b.col(T.INT, 0, False)
    b.count().sum(idc)
    (cnt, total), = _run(capi.Plan(gpu_api, b.build()), [], store)
    assert cnt == (n * 9) // 10
    assert total == int(survivors.sum()) + n * (len(survivors) - 1)
    b = PlanBuilder()
    idc, st = b.col(T.INT, 0, False), b.col(T.BOOLEAN, 1, False)
    b.filter(idc.eq(b.lit(T.INT)))
    b.count().max(idc).count(st)
    pq = capi.Plan(gpu_api, b.build())
    assert _run(pq, [73], store) == [[1, 73, 1]]
    assert _run(pq, [74], store)[0][0] == 0
    # BOOLEAN target: SD_ERR_UNSUPPORTED, nothing installed
    before = [store.get_delta(i, 0, 0) for i in range(5)], [store.get_deletes(i) for i in range(5)]
    b = PlanBuilder()
    s = b.col(T.BOOLEAN, 1)
    b.update({1: s})
    with pytest.raises(SdError) as e:
        capi.Plan(gpu_api, b.build()).update_store(store, [])
    assert e.value.code == capi.SD_ERR_UNSUPPORTED
    assert ([store.get_delta(i, 0, 0) for i in range(5)], [store.get_deletes(i) for i in range(5)]) == before
    assert _run(pq, [73], store) == [[1, 73, 1]]
    store.close()


# ---- nullable narrow-width targets -------------------------------------------------------------------------------------------
NSCHEMA = [(T.INT, False), (T.INT, True), (T.SHORT, True), (T.FLOAT, True), (T.BYTE, True), (T.LONG, True)]
NP = {T.INT: np.int32, T.SHORT: np.int16, T.FLOAT: np.float32, T.BYTE: np.int8, T.LONG: np.int64}


def test_nullable_narrow_targets_bytes_over_two_statements(gpu_api):
    rng = np.random.default_rng(9)
    nrows, nb = 5000, 3
    store = capi.Store(gpu_api, NSCHEMA)
    vals, nulls, d0 = [], [], []
    for bi in range(nb):
        ids = np.arange(bi * nrows, (bi + 1) * nrows, dtype=np.int32)
        v = {0: ids, 1: rng.integers(-10**9, 10**9, nrows).astype(np.int32), 2: rng.integers(-1000, 1000, nrows).astype(np.int16),
             3: (rng.integers(-10**6, 10**6, nrows) / 64.0).astype(np.float32), 4: rng.integers(-60, 60, nrows).astype(np.int8),
             5: rng.integers(-10**12, 10**12, nrows).astype(np.int64)}
        nl = {c: (rng.random(nrows) < 0.1) for c in range(1, 6)}
        cols = [encode_uncompressed(v[0], T.INT)] + [encode_uncompressed(v[c], NSCHEMA[c][0], nl[c]) for c in range(1, 6)]
        cs = [column_stats(v[0], T.INT)] + [column_stats(v[c], NSCHEMA[c][0], nl[c]) for c in range(1, 6)]
        delta0 = {}
        if bi == 0:   # existing Uncompressed depth-0 delta of v with NULLs
            pos = np.sort(rng.choice(nrows, 400, replace=False)).astype(np.int32)
            nv, nn = rng.integers(-100, 100, 400).astype(np.int32), rng.random(400) < 0.3
            delta0[1] = encode_delta(nrows, pos, nv, T.INT, nn)
            v[1][pos], nl[1][pos] = nv, nn
        if bi == 1:   # existing Dictionary-encoded depth-0 delta of the LONG column with NULLs
            pos = np.sort(rng.choice(nrows, 300, replace=False)).astype(np.int32)
            nv, nn = rng.choice(np.array([7, -9, 10**11], dtype=np.int64), 300), rng.random(300) < 0.2
            delta0[5] = encode_delta(nrows, pos, nv, T.LONG, nn, dictionary=True)
            v[5][pos], nl[5][pos] = nv, nn
        store.put(ColumnBatch(num_rows=nrows, columns=cols, stats=stats_row(nrows, cs, has_deltas=bool(delta0)), delta0=delta0, batch_id=bi))
        vals.append(v)
        nulls.append(nl)
        d0.append(dict(delta0))

    def statement(plan, lits, lo, hi, new_fn):
        old_stats = [parse_unsafe_row(store.get_stats(i), _stats_types()) for i in range(nb)]
        rows = plan.update_store(store, lits)
        total = 0
        for bi in range(nb):
            sel = (vals[bi][0] >= lo) & (vals[bi][0] < hi)
            pos = np.nonzero(sel)[0].astype(np.int32)
            total += len(pos)
            if not len(pos):
                assert parse_unsafe_row(store.get_stats(bi), _stats_types()) == old_stats[bi]
                continue
            news = {c: f(bi, pos) for c, f in new_fn.items()}   # SET values read the row as it was before the statement
            exp_stats = list(old_stats[bi])
            exp_stats[0] = -abs(exp_stats[0])
            for c, (nv, nn) in news.items():
                t = NSCHEMA[c][0]
                enc = encode_delta(nrows, pos, nv, t, nn)
                d0[bi][c] = _merge(gpu_api, t, True, enc, d0[bi][c], nrows) if c in d0[bi] else enc
                vals[bi][c][pos], nulls[bi][c][pos] = nv, nn
                f = 1 + 3 * c   # ColumnDelta.mergeStats restated
                nonnull = nv[~nn]
                if len(nonnull):
                    exp_stats[f] = nonnull.min().item() if exp_stats[f] is None else min(exp_stats[f], nonnull.min().item())
                    exp_stats[f + 1] = nonnull.max().item() if exp_stats[f + 1] is None else max(exp_stats[f + 1], nonnull.max().item())
                old_nc = old_stats[bi][f + 2]
                nc = max(old_nc - (len(pos) - int(nn.sum())), int(nn.sum()))
                exp_stats[f + 2] = 1 if nc <= 0 and old_nc > 0 else nc
            for c in range(1, 6):
                if c in d0[bi]:
                    assert store.get_delta(bi, c, 0) == d0[bi][c], (bi, c)
            got = parse_unsafe_row(store.get_stats(bi), _stats_types())
            assert got == exp_stats, bi
        assert rows == total

    b = PlanBuilder()
    c = [b.col(t, i, n) for i, (t, n) in enumerate(NSCHEMA)]
    b.filter((c[0] >= b.lit(T.INT)) & (c[0] < b.lit(T.INT)))
    b.update({1: c[1] + b.lit(T.INT), 2: c[2] + c[2], 3: c[3] + c[3], 4: c[4], 5: c[5] + b.lit(T.LONG)})
    p1 = capi.Plan(gpu_api, b.build())
    with np.errstate(over="ignore"):
        statement(p1, [1000, 12000, 1, 3], 1000, 12000, {
            1: lambda bi, pos: ((vals[bi][1][pos] + np.int32(1)).astype(np.int32), nulls[bi][1][pos].copy()),
            2: lambda bi, pos: ((vals[bi][2][pos] + vals[bi][2][pos]).astype(np.int16), nulls[bi][2][pos].copy()),
            3: lambda bi, pos: ((vals[bi][3][pos] + vals[bi][3][pos]).astype(np.float32), nulls[bi][3][pos].copy()),
            4: lambda bi, pos: (vals[bi][4][pos].copy(), nulls[bi][4][pos].copy()),
            5: lambda bi, pos: ((vals[bi][5][pos] + np.int64(3)).astype(np.int64), nulls[bi][5][pos].copy())})
    b = PlanBuilder()   # second statement, overlapping the first: v = NULL, the LONG column shifted again
    c = [b.col(t, i, n) for i, (t, n) in enumerate(NSCHEMA)]
    b.filter((c[0] >= b.lit(T.INT)) & (c[0] < b.lit(T.INT)))
    b.update({1: b.lit(T.INT), 5: c[5] - b.lit(T.LONG)})
    p2 = capi.Plan(gpu_api, b.build())
    statement(p2, [8000, 15000, None, 5], 8000, 15000, {
        1: lambda bi, pos: (np.zeros(len(pos), np.int32), np.ones(len(pos), bool)),
        5: lambda bi, pos: ((vals[bi][5][pos] - np.int64(5)).astype(np.int64), nulls[bi][5][pos].copy())})
    # the scan over the merged deltas (overlay path with NULLs) sees the effective values
    b = PlanBuilder()
    c = [b.col(t, i, n) for i, (t, n) in enumerate(NSCHEMA)]
    b.count(c[1]).sum(c[1]).sum(c[2]).sum(c[3]).sum(c[5]).count(c[4])
    got, = _run(capi.Plan(gpu_api, b.build()), [], store)
    want = [0, 0, 0, 0.0, 0, 0]
    for bi in range(nb):
        v, nl = vals[bi], nulls[bi]
        want[0] += int((~nl[1]).sum())
        want[1] += int(v[1][~nl[1]].astype(np.int64).sum())
        want[2] += int(v[2][~nl[2]].astype(np.int64).sum())
        want[3] += float(v[3][~nl[3]].astype(np.float64).sum())
        want[4] += int(v[5][~nl[5]].sum())
        want[5] += int((~nl[4]).sum())
    assert got[:3] == want[:3] and got[4:] == want[4:] and got[3] == pytest.approx(want[3], rel=1e-9)
    store.close()


def _stats_types():
    return [T.INT] + [t for tt, _ in NSCHEMA for t in (tt, tt, T.INT)]


# ---- batches appended while statements run ----------------------------------------------------------------------------------
def test_batches_appended_during_updates_stay_untouched(gpu_api):
    rpb, nb0, nstmt = 50_000, 8, 6
    store = capi.Store(gpu_api, lineitem.LINEITEM_SCHEMA)
    store.gen_lineitem(0, nb0 * rpb, rpb, 4, 3, lineitem.Q6_COLUMN_MASK)
    b = PlanBuilder()
    q = b.col(T.DOUBLE, L_QUANTITY)
    b.update({L_QUANTITY: q + b.lit(T.DOUBLE)})
    up = capi.Plan(gpu_api, b.build())
    errors, done = [], threading.Event()

    def ingest():
        try:
            gpu_api.check(gpu_api.init(0))
            k = nb0
            while not done.is_set() and k < nb0 + 40:
                store.gen_lineitem(k * rpb, rpb, rpb, 4, 3, lineitem.Q6_COLUMN_MASK)
                k += 1
        except Exception as e:   # reported below
            errors.append(e)

    t = threading.Thread(target=ingest)
    t.start()
    rows = [up.update_store(store, [1.0]) for _ in range(nstmt)]
    done.set()
    t.join()
    assert not errors, errors
    nb = store.num_batches()
    ks = []
    for i in range(nb):
        nrows, _, _ = store.batch_info(i)
        base = lineitem.lineitem_values(i * rpb, nrows, 3)["l_quantity"]
        try:
            d = store.get_delta(i, L_QUANTITY, 0)
        except SdError:
            ks.append(0)
            continue
        nbw, = struct.unpack_from("<i", d, 4)
        n, = struct.unpack_from("<i", d, 12 + nbw)
        body = ((8 + nbw + 8 + 4 * n + 7) // 8) * 8
        assert n == nrows
        k = np.frombuffer(d, dtype="<f8", count=n, offset=body) - base
        assert np.all(k == k[0]) and k[0] == round(k[0]), i   # a statement updates a batch whole or not at all
        ks.append(int(k[0]))
    assert ks[:nb0] == [nstmt] * nb0
    assert all(ks[i] >= ks[i + 1] for i in range(nb - 1)), ks   # a batch appended later saw no more statements than an older one
    rows_per = [store.batch_info(i)[0] for i in range(nb)]
    assert sum(rows) == sum(k * r for k, r in zip(ks, rows_per))
    store.close()


# ---- at scale: the staged ring wraps ----------------------------------------------------------------------------------------
def test_one_percent_update_and_delete_over_60m_rows(gpu_api):
    total, rpb, seed = 59_986_052, 200_000, 6
    store = capi.Store(gpu_api, lineitem.LINEITEM_SCHEMA)
    store.gen_lineitem(0, total, rpb, 128, seed, lineitem.Q6_COLUMN_MASK)
    nb = store.num_batches()
    b = PlanBuilder()
    disc, ship = b.col(T.DOUBLE, L_DISCOUNT), b.col(T.DATE, L_SHIPDATE)
    b.filter(ship <= b.lit(T.DATE))
    b.update({L_DISCOUNT: disc + b.lit(T.DOUBLE)})
    rows_u = capi.Plan(gpu_api, b.build()).update_store(store, [8061, 0.01])   # 26 of 2526 ship dates: ~1 %
    b = PlanBuilder()
    ship = b.col(T.DATE, L_SHIPDATE)
    b.filter((ship >= b.lit(T.DATE)) & (ship < b.lit(T.DATE)))
    b.delete()
    rows_d = capi.Plan(gpu_api, b.build()).delete_store(store, [8100, 8126])
    want_u = want_d = 0
    for i in range(nb):
        nrows, _, _ = store.batch_info(i)
        v = lineitem.lineitem_values(i * rpb, nrows, seed)
        pos = np.nonzero(v["l_shipdate"] <= 8061)[0].astype(np.int32)
        want_u += len(pos)
        assert store.get_delta(i, L_DISCOUNT, 0) == encode_delta(nrows, pos, v["l_discount"][pos] + 0.01, T.DOUBLE), i
        dpos = np.nonzero((v["l_shipdate"] >= 8100) & (v["l_shipdate"] < 8126))[0].astype(np.int32)
        want_d += len(dpos)
        assert store.get_deletes(i) == encode_delete(nrows, dpos), i
    assert (rows_u, rows_d) == (want_u, want_d)
    assert 0.008 * total < rows_u < 0.012 * total
    store.close()
