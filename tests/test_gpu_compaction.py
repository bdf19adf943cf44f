"""Compaction on the device (sd_store_compact): the update deltas and delete masks of resident batches folded back into their
base columns.  A rewritten column's bytes are the fixture writer's default encoding of the batch's live rows with their
current values -- and what sd_store_encode_batch writes for them in another store; kept columns keep their bytes; query results
do not move (against numpy and against the CPU oracle over host ColumnBatches rebuilt from the compacted bytes); the selection
threshold; fully deleted batches leave the store; later statements address the renumbered rows; refusals leave the store as it
was; a concurrent reader sees all of a compaction or none; the staged fast path is back afterwards."""
import math
import struct
import threading

import numpy as np
import pytest

from snappydata_b200 import capi, lineitem, plan as P
from snappydata_b200.capi import SdError
from snappydata_b200.column_format import (ColumnBatch, SqlType as T, compress_lz4, decode_column, encode_column, encode_delete,
                                           encode_delta, encode_dictionary, encode_run_length, encode_uncompressed, parse_unsafe_row)
from snappydata_b200.plan import L_DISCOUNT, L_QUANTITY, L_SHIPDATE, PlanBuilder

import known_answer_cases as K
from helpers import assert_rowsets_match
from test_gpu_mutations import NB, RPB, Model, _update_plan

pytestmark = pytest.mark.gpu

RESIDENT = (L_QUANTITY, P.L_EXTENDEDPRICE, L_DISCOUNT, P.L_TAX, P.L_RETURNFLAG, P.L_LINESTATUS, L_SHIPDATE)
STATS_TYPES = [T.INT] + [t for c in range(16) for t in (lineitem.LINEITEM_SCHEMA[c][0],) * 2 + (T.INT,)]


def _typ(c):
    return lineitem.LINEITEM_SCHEMA[c][0]


class Table:
    """Model of test_gpu_mutations plus every resident column's current values, restated in numpy at every step."""

    def __init__(self, api):
        self.m = Model(np.random.default_rng(3), api)
        self.store = capi.Store(api, lineitem.LINEITEM_SCHEMA)
        for b in self.m.batches:
            self.store.put(b)
        self.cur = []   # per batch: {col: current values of every base row}
        for i, b in enumerate(self.m.batches):
            v = {c: decode_column(b.columns[c], _typ(c), b.num_rows)[0] for c in RESIDENT}
            v.update(self.m.vals[i])
            self.cur.append(v)
        self.live = [l.copy() for l in self.m.live]
        self.dirty = [bool(self.m.delta0[i] or self.m.delta1[i] or self.m.mask[i] is not None) for i in range(NB)]
        self.delta_cols = [set(self.m.delta0[i]) | set(self.m.delta1[i]) for i in range(NB)]

    def live_values(self, i, c):
        return self.cur[i][c][self.live[i]]

    def compacted(self, i):
        """After a compaction: batch i holds only its live rows, renumbered from 0."""
        self.cur[i] = {c: v[self.live[i]] for c, v in self.cur[i].items()}
        self.live[i] = np.ones(len(self.cur[i][L_QUANTITY]), bool)
        self.dirty[i] = False

    def q6(self):
        d0, d1, lo, hi, q = P.Q6_LITERALS
        want = 0.0
        for i in range(len(self.cur)):
            v = self.cur[i]
            sel = self.live[i] & (v[L_SHIPDATE] >= d0) & (v[L_SHIPDATE] < d1) & (v[L_DISCOUNT] >= lo) & (v[L_DISCOUNT] <= hi) & (v[L_QUANTITY] < q)
            want += float(np.sum(v[P.L_EXTENDEDPRICE][sel] * v[L_DISCOUNT][sel]))
        return want


@pytest.fixture()
def tab(gpu_api):
    t = Table(gpu_api)
    yield t
    t.store.close()


def _q(gp, store, lits):
    return capi.parse_row_stream(gp.execute_store_raw(store, gp.literal_array(lits), len(lits)), gp.desc.partial_schema())


def _statements(gpu_api, t):
    """An UPDATE and a DELETE through the device path, restated in numpy."""
    up = capi.Plan(gpu_api, _update_plan(lambda b, c: {L_DISCOUNT: c[L_DISCOUNT] + b.lit(T.DOUBLE), L_QUANTITY: b.lit(T.DOUBLE)},
                                         lambda b, c: (c[L_SHIPDATE] >= b.lit(T.DATE)) & (c[L_SHIPDATE] <= b.lit(T.DATE))))
    rows = up.update_store(t.store, [8800, 9100, 0.01, 7.0])
    n = 0
    for i in range(NB):
        v = t.cur[i]
        sel = t.live[i] & (v[L_SHIPDATE] >= 8800) & (v[L_SHIPDATE] <= 9100)
        n += int(sel.sum())
        v[L_DISCOUNT] = np.where(sel, v[L_DISCOUNT] + 0.01, v[L_DISCOUNT])
        v[L_QUANTITY] = np.where(sel, 7.0, v[L_QUANTITY])
        t.dirty[i] |= bool(sel.any())
        if sel.any():
            t.delta_cols[i] |= {L_DISCOUNT, L_QUANTITY}
    assert rows == n
    dp = capi.Plan(gpu_api, _update_plan(None, lambda b, c: c[L_QUANTITY] < b.lit(T.DOUBLE)))
    rows = dp.delete_store(t.store, [4.0])
    n = 0
    for i in range(NB):
        sel = t.live[i] & (t.cur[i][L_QUANTITY] < 4.0)
        n += int(sel.sum())
        t.live[i] &= ~sel
        t.dirty[i] |= bool(sel.any())
    assert rows == n
    up.close()
    dp.close()


@pytest.mark.parametrize("round_bytes", [None, "1"])   # "1": every batch is a round of its own
def test_compacted_bytes_stats_and_query_results(gpu_api, tab, monkeypatch, round_bytes):
    from oracle import oracle
    t, store = tab, tab.store
    if round_bytes:
        monkeypatch.setenv("SD_TUNE_COMPACT_ROUND_BYTES", round_bytes)
    _statements(gpu_api, t)
    old_stats = [parse_unsafe_row(store.get_stats(i), STATS_TYPES) for i in range(NB)]
    plans = [(d, l, k, capi.Plan(gpu_api, d)) for d, l, k in ((P.q6_plan(), P.Q6_LITERALS, 0), (P.q1_plan(), P.Q1_LITERALS, 2))]
    before = [_q(gp, store, l) for _, l, _, gp in plans]
    old = {(i, c): store.get_buffer(i, c) for i in range(NB) for c in RESIDENT}
    masked = [i for i in range(NB) if not t.live[i].all() or t.m.mask[i] is not None]
    res = store.compact(0.0)
    assert res["batches_rewritten"] == sum(t.dirty) and res["batches_removed"] == 0
    assert res["rows_purged"] == sum(int((~l).sum()) for l in t.live) and res["bytes_written"] > 0
    tm = capi.last_compaction_timing(gpu_api)
    assert tm["materialise_ms"] > 0 and tm["bytes_read"] > 0
    ref = capi.Store(gpu_api, lineitem.LINEITEM_SCHEMA)   # the same live rows through ingest
    for i in range(NB):
        ref.encode_batch(int(t.live[i].sum()), {c: (t.live_values(i, c), None) for c in RESIDENT}, t.m.batches[i].bucket_id,
                         t.m.batches[i].batch_id)
    for i in range(NB):
        assert store.batch_info(i) == (int(t.live[i].sum()), t.m.batches[i].bucket_id, t.m.batches[i].batch_id)
        if not t.dirty[i]:
            assert all(store.get_buffer(i, c) == old[(i, c)] for c in RESIDENT)
            continue
        st, rst = parse_unsafe_row(store.get_stats(i), STATS_TYPES), parse_unsafe_row(ref.get_stats(i), STATS_TYPES)
        assert st[0] == int(t.live[i].sum())
        for c in range(16):   # the entries of the columns that were not rewritten stay as they were
            if c not in RESIDENT or not (i in masked or c in t.delta_cols[i]):
                assert st[1 + 3 * c: 4 + 3 * c] == old_stats[i][1 + 3 * c: 4 + 3 * c], (i, c)
        for c in RESIDENT:
            got = store.get_buffer(i, c)
            if i in masked or c in t.delta_cols[i]:
                assert got == encode_column(t.live_values(i, c), _typ(c)), (i, c)
                assert got == ref.get_buffer(i, c), (i, c)
                assert st[1 + 3 * c: 4 + 3 * c] == rst[1 + 3 * c: 4 + 3 * c], (i, c)
            else:
                assert got == old[(i, c)], (i, c)
            for depth in (0, 1):
                with pytest.raises(SdError):
                    store.get_delta(i, c, depth)
        with pytest.raises(SdError):
            store.get_deletes(i)
    # query results: exact counts, doubles to 1e-6 (batch sizes change the reduction order); the oracle over the new bytes
    for (desc, lits, nkeys, gp), b4 in zip(plans, before):
        got = _q(gp, store, lits)
        assert_rowsets_match(got, b4, nkeys)
        op = oracle.plan(desc).set_literals(lits)
        for i in range(NB):
            n, bucket, bid = store.batch_info(i)
            cols = [None] * 16
            for c in RESIDENT:
                cols[c] = store.get_buffer(i, c)
            op.submit(ColumnBatch(num_rows=n, columns=cols, batch_id=bid, bucket_id=bucket))
        assert_rowsets_match(got, op.finish(), nkeys)
        op.close()
        m = gp.metrics()
        assert m["updatedColumnCount"] == 0 and m["deletedBatchCount"] == 0
    (q6,), = _q(plans[0][3], store, P.Q6_LITERALS)
    assert q6 == pytest.approx(t.q6(), rel=1e-6)
    # the staged fast path: as many algorithmic bytes as a store encoded fresh from the same rows
    fresh = capi.Plan(gpu_api, P.q1_plan())
    _q(fresh, ref, P.Q1_LITERALS)
    assert plans[1][3].metrics()["algorithmicBytes"] == fresh.metrics()["algorithmicBytes"]
    for p in plans:
        p[3].close()
    fresh.close()
    ref.close()


def test_selection_threshold(gpu_api, tab):
    t, store = tab, tab.store
    frac = []
    for i in range(NB):
        d = sum(struct.unpack_from("<ii", t.m.delta0[i][c], 8 + struct.unpack_from("<i", t.m.delta0[i][c], 4)[0])[1] for c in t.m.delta0[i])
        d += sum(struct.unpack_from("<ii", t.m.delta1[i][c], 8 + struct.unpack_from("<i", t.m.delta1[i][c], 4)[0])[1] for c in t.m.delta1[i])
        d += int((~t.live[i]).sum())
        frac.append(d / RPB)
    dirty = sorted({f for f in frac if f > 0})
    assert len(dirty) >= 2
    thr = (dirty[0] + dirty[1]) / 2
    bufs = [store.get_buffer(i, L_QUANTITY) for i in range(NB)]
    res = store.compact(thr)
    assert res["batches_rewritten"] == sum(f >= thr for f in frac)
    for i in range(NB):
        if frac[i] >= thr:
            assert store.batch_info(i)[0] == int(t.live[i].sum())
            with pytest.raises(SdError):
                store.get_deletes(i) if t.m.mask[i] is not None else store.get_delta(i, L_QUANTITY, 0)
        else:
            assert store.get_buffer(i, L_QUANTITY) == bufs[i]
            for c in t.m.delta0[i]:
                assert store.get_delta(i, c, 0) == t.m.delta0[i][c]
            if t.m.mask[i] is not None:
                assert store.get_deletes(i) == t.m.mask[i]


def test_fully_deleted_batch_leaves_the_store(gpu_api, tab):
    t, store = tab, tab.store
    dp = capi.Plan(gpu_api, _update_plan(None, lambda b, c: None))
    ids = [store.batch_info(i)[2] for i in range(NB)]
    gone = [i for i in range(NB) if t.m.batches[i].bucket_id == 1]
    dp.delete_store(store, [], buckets=[1])
    q6 = capi.Plan(gpu_api, P.q6_plan())
    before = _q(q6, store, P.Q6_LITERALS)
    res = store.compact(0.0)
    assert res["batches_removed"] == len(gone)
    assert store.num_batches() == NB - len(gone)
    assert [store.batch_info(i)[2] for i in range(store.num_batches())] == [ids[i] for i in range(NB) if i not in gone]
    (a,), (b,) = before[0], _q(q6, store, P.Q6_LITERALS)[0]
    assert b == pytest.approx(a, rel=1e-6)
    dp.close()
    q6.close()


def test_later_statements_address_the_new_ordinals(gpu_api, tab):
    t, store = tab, tab.store
    up = capi.Plan(gpu_api, _update_plan(lambda b, c: {L_QUANTITY: c[L_QUANTITY] + b.lit(T.DOUBLE)},
                                         lambda b, c: c[L_SHIPDATE] < b.lit(T.DATE)))
    dp = capi.Plan(gpu_api, _update_plan(None, lambda b, c: c[L_DISCOUNT] > b.lit(T.DOUBLE)))
    q6 = capi.Plan(gpu_api, P.q6_plan())

    def update(k, add):
        rows = up.update_store(store, [k, add])
        n = 0
        for i in range(len(t.cur)):
            sel = t.live[i] & (t.cur[i][L_SHIPDATE] < k)
            n += int(sel.sum())
            t.cur[i][L_QUANTITY] = np.where(sel, t.cur[i][L_QUANTITY] + add, t.cur[i][L_QUANTITY])
            t.dirty[i] |= bool(sel.any())
        assert rows == n

    def compact():
        store.compact(0.0)
        dirty = [i for i in range(NB) if t.dirty[i]]
        for i in dirty:
            t.compacted(i)
        for i in dirty:
            for c in RESIDENT:
                assert store.get_buffer(i, c) == encode_column(t.live_values(i, c), _typ(c)), (i, c)
        (got,), = _q(q6, store, P.Q6_LITERALS)
        assert got == pytest.approx(t.q6(), rel=1e-6)

    update(8500, 1.0)
    compact()
    update(9000, 2.0)
    rows = dp.delete_store(store, [0.08])
    n = 0
    for i in range(NB):
        sel = t.live[i] & (t.cur[i][L_DISCOUNT] > 0.08)
        n += int(sel.sum())
        t.live[i] &= ~sel
        t.dirty[i] |= bool(sel.any())
    assert rows == n
    compact()
    for p in (up, dp, q6):
        p.close()


# ---- every base encoding x type x nullability -----------------------------------------------------------------------------------
N = 3000
CASES = [("uncompressed", T.INT, True), ("uncompressed", T.SHORT, True), ("uncompressed", T.BYTE, True), ("uncompressed", T.FLOAT, True),
         ("uncompressed", T.LONG, True), ("uncompressed", T.DOUBLE, False), ("dictionary", T.INT, True), ("dictionary", T.LONG, False),
         ("dictionary", T.STRING, True), ("dictionary", T.STRING, False), ("runlength", T.INT, True), ("runlength", T.STRING, False),
         ("bitset", T.BOOLEAN, True), ("lz4", T.INT, True), ("lz4", T.STRING, True)]


def _vals(t, r, m):
    if t == T.STRING:
        return np.array([b"k%d" % x for x in r.integers(0, 30, m)], dtype=object)
    if t == T.BOOLEAN:
        return r.integers(0, 2, m).astype(bool)
    if t in (T.FLOAT, T.DOUBLE):
        return np.round(r.normal(0, 40, m), 2).astype(np.float32 if t == T.FLOAT else np.float64)
    return np.repeat(r.integers(-100, 100, m // 10 + 1), 10)[:m] if m > 20 else r.integers(-100, 100, m)


@pytest.mark.parametrize("enc,t,nullable", CASES)
@pytest.mark.parametrize("shape", ["deltas", "deletes", "both"])
def test_every_base_encoding(gpu_api, enc, t, nullable, shape):
    r = np.random.default_rng(CASES.index((enc, t, nullable)) * 3 + ["deltas", "deletes", "both"].index(shape))
    base = _vals(t, r, N)
    nulls = (r.random(N) < 0.1) if nullable else None
    col = {"uncompressed": lambda: encode_uncompressed(base, t, nulls), "dictionary": lambda: encode_dictionary(base, t, nulls),
           "runlength": lambda: encode_run_length(base, t, nulls), "bitset": lambda: encode_column(base, t, nulls),
           "lz4": lambda: compress_lz4(encode_column(base, t, nulls) if t == T.STRING else encode_uncompressed(base, t, nulls), force=True)}[enc]()
    eff = np.array(list(base), dtype=object) if t == T.STRING else base.copy()
    eff_n = nulls.copy() if nullable else np.zeros(N, bool)
    other = np.arange(N, dtype=np.int64)
    b = ColumnBatch(num_rows=N, columns=[col, encode_uncompressed(other, T.LONG)], batch_id=4, bucket_id=2)
    if shape in ("deltas", "both"):
        d = {}
        for depth in (1, 0):
            pos = np.sort(r.choice(N, 300, replace=False)).astype(np.int32)
            v = _vals(t, r, 300)
            dn = (r.random(300) < 0.2) if nullable else None
            d[depth] = encode_delta(N, pos, v, t, dn)
            eff[pos] = v
            if nullable:
                eff_n[pos] = dn
        b.delta1, b.delta0 = {0: d[1]}, {0: d[0]}
    live = np.ones(N, bool)
    if shape in ("deletes", "both"):
        dp = np.sort(r.choice(N, 400, replace=False)).astype(np.int32)
        b.delete_mask = encode_delete(N, dp)
        live[dp] = False
    store = capi.Store(gpu_api, [(t, nullable), (T.LONG, False)])
    store.put(b)
    res = store.compact(0.0)
    assert res["batches_rewritten"] == 1
    want = encode_column(eff[live], t, eff_n[live] if nullable else None)
    assert store.get_buffer(0, 0) == want
    other_want = encode_uncompressed(other[live], T.LONG) if shape != "deltas" else encode_uncompressed(other, T.LONG)
    assert store.get_buffer(0, 1) == other_want
    assert store.batch_info(0) == (int(live.sum()), 2, 4)
    store.close()


# ---- refusals -------------------------------------------------------------------------------------------------------------------
def test_refusals_leave_the_store_unchanged(gpu_api, tab):
    t, store = tab, tab.store
    q6 = capi.Plan(gpu_api, P.q6_plan())
    snap = lambda: ([store.get_buffer(i, c) for i in range(NB) for c in RESIDENT], [store.get_stats(i) for i in range(NB)],
                    store.nbytes(), _q(q6, store, P.Q6_LITERALS))
    before = snap()
    for bad in (-0.5, math.nan):
        with pytest.raises(SdError) as e:
            store.compact(bad)
        assert e.value.code == capi.SD_ERR_INVALID
        assert snap() == before
    q6.close()
    # an Uncompressed (variable-width) STRING column in a batch with deletes
    s2 = capi.Store(gpu_api, [(T.STRING, False), (T.INT, False)])
    vals = [b"a%d" % i for i in range(100)]
    s2.put(ColumnBatch(num_rows=100, columns=[encode_uncompressed(vals, T.STRING), encode_uncompressed(np.arange(100), T.INT)],
                       delete_mask=encode_delete(100, [3, 50]), batch_id=9))
    b4 = (s2.get_buffer(0, 0), s2.get_buffer(0, 1), s2.get_deletes(0), s2.nbytes())
    with pytest.raises(SdError) as e:
        s2.compact(0.0)
    assert e.value.code == capi.SD_ERR_UNSUPPORTED and "batch 9" in str(e.value)
    assert (s2.get_buffer(0, 0), s2.get_buffer(0, 1), s2.get_deletes(0), s2.nbytes()) == b4
    s2.close()


# ---- atomicity and concurrency ----------------------------------------------------------------------------------------------------
def test_reader_sees_all_or_nothing_and_ingest_survives(gpu_api, tab):
    t, store = tab, tab.store
    b = PlanBuilder()
    b.count().sum(b.col(T.DOUBLE, L_QUANTITY))
    qdesc = b.build()
    want = (sum(int(l.sum()) for l in t.live), sum(float(t.cur[i][L_QUANTITY][t.live[i]].sum()) for i in range(NB)))
    seen, stop, running, errors = [], threading.Event(), threading.Event(), []

    def reader():
        try:
            gpu_api.check(gpu_api.init(0))
            qp = capi.Plan(gpu_api, qdesc)
            while not stop.is_set():
                (cnt, s), = capi.parse_row_stream(qp.execute_store_raw(store, qp.literal_array([]), 0), qdesc.partial_schema())
                seen.append((cnt, s))
                running.set()
            qp.close()
        except Exception as e:   # reported below
            errors.append(e)
            running.set()

    extra = [(5, np.full(5, 3.0)), (7, np.full(7, 4.0))]

    def ingest():
        try:
            gpu_api.check(gpu_api.init(0))
            for k, (n, q) in enumerate(extra):
                store.encode_batch(n, {L_QUANTITY: (q, None), L_SHIPDATE: (np.full(n, 9000, np.int32), None)}, 9, 1000 + k)
        except Exception as e:
            errors.append(e)

    rt, it = threading.Thread(target=reader), threading.Thread(target=ingest)
    rt.start()
    running.wait()   # the reader's plan is built and it is querying
    it.start()
    n0 = len(seen)
    store.compact(0.0)
    it.join()
    while len(seen) < n0 + 3 and not errors:   # a few queries after the compaction
        running.clear()
        running.wait()
    stop.set()
    rt.join()
    assert not errors, errors
    allowed = {want}
    for k in range(len(extra) + 1):
        allowed.add((want[0] + sum(n for n, _ in extra[:k]), want[1] + sum(float(q.sum()) for _, q in extra[:k])))
    assert set(seen) <= allowed, (set(seen), allowed)
    assert seen[-1] == max(allowed)
    ids = [store.batch_info(i)[2] for i in range(store.num_batches())]
    assert 1000 in ids and 1001 in ids and store.num_batches() == NB + 2
    assert store.get_buffer(ids.index(1001), L_QUANTITY) == encode_column(np.full(7, 4.0), T.DOUBLE)


def test_update_and_compaction_from_two_threads_serialise(gpu_api, tab):
    t, store = tab, tab.store
    up = capi.Plan(gpu_api, _update_plan(lambda b, c: {L_QUANTITY: c[L_QUANTITY] + b.lit(T.DOUBLE)}, lambda b, c: None))
    errors = []

    def upd():
        try:
            gpu_api.check(gpu_api.init(0))
            up.update_store(store, [1.0])
        except Exception as e:
            errors.append(e)

    th = threading.Thread(target=upd)
    th.start()
    store.compact(0.0)
    th.join()
    assert not errors, errors
    # whichever order ran, the current values are the restatement's; a final compaction leaves exactly them
    for i in range(NB):
        t.cur[i][L_QUANTITY] = t.cur[i][L_QUANTITY] + 1.0
    store.compact(0.0)
    for i in range(NB):
        t.compacted(i)
        assert store.get_buffer(i, L_QUANTITY) == encode_column(t.live_values(i, L_QUANTITY), T.DOUBLE), i
    up.close()


# ---- the reference's closed forms with a compaction in between -----------------------------------------------------------------
def _compacting_runner(api, schema):
    def run(desc, lits, batches):
        store = capi.Store(api, schema)
        for b in batches:
            store.put(b)
        store.compact(0.0)
        assert store.num_batches() == len(batches)
        p = capi.Plan(api, desc)
        rows = capi.parse_row_stream(p.execute_store_raw(store, p.literal_array(lits), len(lits)), desc.partial_schema())
        p.close()
        store.close()
        return (rows,)
    return run


def test_known_answers_survive_compaction(gpu_api):
    K.case_delta_stats_point_filters_after_updates(_compacting_runner(gpu_api, [(T.LONG, False), (T.LONG, False)]))
    K.case_basic_delete_and_update_counts(_compacting_runner(gpu_api, [(T.INT, False), (T.BOOLEAN, False)]))


# ---- scale: a 60 M-row store, 1 % UPDATE + 1 % DELETE, compaction over several rounds ----------------------------------------
def test_compaction_over_60m_rows(gpu_api):
    from oracle import oracle
    total, rpb, seed = 59_986_052, 200_000, 6
    store = capi.Store(gpu_api, lineitem.LINEITEM_SCHEMA)
    store.gen_lineitem(0, total, rpb, 128, seed, lineitem.Q1_COLUMN_MASK)
    nb = store.num_batches()
    b = PlanBuilder()
    disc, ship = b.col(T.DOUBLE, L_DISCOUNT), b.col(T.DATE, L_SHIPDATE)
    b.filter(ship <= b.lit(T.DATE))
    b.update({L_DISCOUNT: disc + b.lit(T.DOUBLE)})
    up = capi.Plan(gpu_api, b.build())
    rows_u = up.update_store(store, [8061, 0.01])   # 26 of 2526 ship dates: ~1 %
    b = PlanBuilder()
    ship = b.col(T.DATE, L_SHIPDATE)
    b.filter((ship >= b.lit(T.DATE)) & (ship < b.lit(T.DATE)))
    b.delete()
    dp = capi.Plan(gpu_api, b.build())
    rows_d = dp.delete_store(store, [8100, 8126])
    assert 0.008 * total < rows_u < 0.012 * total and 0.008 * total < rows_d < 0.012 * total
    q1 = capi.Plan(gpu_api, P.q1_plan())
    before = _q(q1, store, P.Q1_LITERALS)
    res = store.compact(0.0)   # ~3 GB of materialised values: more than one round of 2 GB
    assert res["batches_rewritten"] == nb and res["batches_removed"] == 0 and res["rows_purged"] == rows_d
    names = {L_QUANTITY: "l_quantity", P.L_EXTENDEDPRICE: "l_extendedprice", L_DISCOUNT: "l_discount", P.L_TAX: "l_tax",
             L_SHIPDATE: "l_shipdate", P.L_RETURNFLAG: "l_returnflag", P.L_LINESTATUS: "l_linestatus"}
    numeric = [c for c in RESIDENT if _typ(c) != T.STRING]
    ref = capi.Store(gpu_api, lineitem.LINEITEM_SCHEMA)   # numpy's live rows re-encoded on the device
    op = oracle.plan(P.q1_plan()).set_literals(P.Q1_LITERALS)
    for i in range(nb):
        nrows = min(rpb, total - i * rpb)
        v = lineitem.lineitem_values(i * rpb, nrows, seed)
        v["l_discount"] = np.where(v["l_shipdate"] <= 8061, v["l_discount"] + 0.01, v["l_discount"])
        live = ~((v["l_shipdate"] >= 8100) & (v["l_shipdate"] < 8126))
        n_live = int(live.sum())
        _, bucket, bid = store.batch_info(i)
        assert store.batch_info(i)[0] == n_live
        ref.encode_batch(n_live, {c: (v[names[c]][live], None) for c in numeric}, bucket, bid)
        cols = [None] * 16
        for c in RESIDENT:
            cols[c] = store.get_buffer(i, c)
            want = ref.get_buffer(i, c) if c in numeric else encode_dictionary(v[names[c]][live], T.STRING)
            assert cols[c] == want, (i, c)
        op.submit(ColumnBatch(num_rows=n_live, columns=cols, batch_id=bid, bucket_id=bucket))
    got = _q(q1, store, P.Q1_LITERALS)
    assert_rowsets_match(got, op.finish(), 2)
    assert_rowsets_match(got, before, 2)
    assert q1.metrics()["updatedColumnCount"] == 0 and q1.metrics()["deletedBatchCount"] == 0
    op.close()
    for p in (up, dp, q1):
        p.close()
    ref.close()
    store.close()
