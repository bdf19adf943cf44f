"""Reclaiming the device memory of superseded batch versions (sd_store_reclaim).

Every kind of allocation a batch version owns -- the column buffers of every encoding, LZ4 destinations, raw-string
positions, null words and their prefixes, run ends, update deltas from puts and from statements with their DevDelta structs,
delete masks, compacted columns -- moves with reclaim(1.0) while every byte the store reports and every query result stays
exactly what it was, for plan handles that ran before and for fresh ones; dead slabs are freed without a copy; memory stays
bounded under repeated UPDATE -> compaction -> reclaim; an unfinished scan pins what it may read; reclaims run beside
queries and ingest; later statements work on moved batches; compression survives; bad arguments are refused."""
import math
import threading

import numpy as np
import pytest

from snappydata_b200 import capi, lineitem, plan as P
from snappydata_b200.capi import AggFn, SdError
from snappydata_b200.column_format import (ColumnBatch, SqlType as T, build_batch, compress_lz4, encode_column)
from snappydata_b200.plan import L_DISCOUNT, L_QUANTITY, L_SHIPDATE, PlanBuilder

import kernel_cases as kc
from helpers import assert_rowsets_match
from test_gpu_compaction import RESIDENT, Table, _q, _statements, _typ
from test_gpu_mutations import NB

pytestmark = pytest.mark.gpu

STORE_SCHEMA = [(t, n) for _, t, n in kc.SCHEMA]
N = 3 * 2048 + 77
DENSE = kc.Query(["k"], kc.EVERY_AGG, filter_lit=-900)                                   # dictionary STRING key
HASH = kc.Query(["h"], [(AggFn.COUNT_STAR, None), (AggFn.SUM, "d"), (AggFn.MIN, "s"), (AggFn.MAX, "s")])   # hash table
NOKEY = kc.Query([], kc.EVERY_AGG)
QUERIES = (DENSE, HASH, NOKEY)


def _run(plan, q, store):
    plan.reset().set_literals(q.literals())
    plan.scan_store(store)
    return capi.parse_row_stream(plan.finish_raw(), q.desc().partial_schema())


def _paths(plan):
    return [(r["paths"], r["accumulator"]) for r in plan.launch_log() if r["replay"] is None]


def _projection():
    b = PlanBuilder()
    e = {n: b.col(kc.TYPE[n], kc.COL[n], kc.NULLABLE[n]) for n in ("k", "s", "i")}
    b.filter(e["i"] > b.lit(T.INT))
    b.project(e["k"], e["s"], e["i"])
    return b.build()


def _rows(plan, store):
    plan.reset().set_literals([500])
    plan.scan_store(store)
    raw = plan.finish_raw()
    out, pos = [], 0
    while pos < len(raw):
        n = int.from_bytes(raw[pos:pos + 8], "little")
        out.append(raw[pos:pos + 8 + n])
        pos += 8 + n
    return sorted(out)


def _snapshot(store):
    """Every byte the store reports about each batch."""
    out = []
    for i in range(store.num_batches()):
        rec = {"info": store.batch_info(i), "stats": store.get_stats(i)}
        for c in range(len(STORE_SCHEMA)):
            try:
                rec[("buf", c)] = store.get_buffer(i, c)
            except SdError:
                rec[("buf", c)] = None
            for depth in (0, 1):
                try:
                    rec[("delta", c, depth)] = store.get_delta(i, c, depth)
                except SdError:
                    rec[("delta", c, depth)] = None
        try:
            rec["deletes"] = store.get_deletes(i)
        except SdError:
            rec["deletes"] = None
        out.append(rec)
    return out


def _identity_update(api):
    """UPDATE t SET d = d WHERE i > -500: the statement merges a device-written depth-0 delta without changing a value."""
    b = PlanBuilder()
    i, d = b.col(T.INT, kc.COL["i"], True), b.col(T.DOUBLE, kc.COL["d"], True)
    b.filter(i > b.lit(T.INT))
    b.update({kc.COL["d"]: d})
    return capi.Plan(api, b.build())


def _delete(api):
    b = PlanBuilder()
    i = b.col(T.INT, kc.COL["i"], True)
    b.filter(i > b.lit(T.INT))
    b.delete()
    return capi.Plan(api, b.build())


def mixed_store(api):
    """One store with every kind of extent; returns (store, raws in store order)."""
    store = capi.Store(api, STORE_SCHEMA)
    raws = []
    bid = 0

    def next_id():   # bucket = batch_id % 4; bucket 3 is kept for the one batch that is compacted
        nonlocal bid
        while bid % 4 == 3:
            bid += 1
        bid += 1
        return bid - 1

    for ki, kind in enumerate(kc.KINDS):
        b, r = kc.make_batch(N, kind, seed=700 + ki, groups=9, batch_id=next_id())
        store.put(b)
        raws.append(r)
    # Uncompressed (variable-width) STRING column
    _, r = kc.make_batch(N, "fast_nulls", seed=720, groups=9)
    i = next_id()
    b = build_batch(N, kc.SCHEMA, r.values, r.nulls, batch_id=i, bucket_id=i % 4, encoders={"s": "uncompressed", "b": "uncompressed"})
    b.stats = None
    store.put(b)
    raws.append(r)
    # LZ4 envelopes, expanded on the device
    b, r = kc.make_batch(N, "fast_nulls", seed=721, groups=9, batch_id=next_id())
    b.columns = [compress_lz4(c, force=True) if c is not None else None for c in b.columns]
    store.put(b)
    raws.append(r)
    # device-encoded
    for seed in (722, 723):
        _, r = kc.make_batch(N, "fast_nulls", seed=seed, groups=9)
        i = next_id()
        store.encode_batch(N, {c: (r.values[name], r.nulls.get(name)) for c, (name, _, _) in enumerate(kc.SCHEMA)}, i % 4, i)
        raws.append(r)
    # the batch to compact: deltas from its put, then a delete mask and a statement's delta
    b, r = kc.make_batch(N, "fast_overlay", seed=724, groups=9, batch_id=3)
    store.put(b)
    raws.append(r)
    # a statement's depth-0 deltas (values unchanged) and delete masks, restated in the raws
    up = _identity_update(api)
    up.update_store(store, [-500])
    dp = _delete(api)
    dp.delete_store(store, [990])
    for r in raws:
        vals, nul = r.effective("i")
        gone = {p for p in range(r.n) if not nul[p] and vals[p] > 990}
        r.deletes = np.array(sorted(set(r.deletes.tolist()) | gone), dtype=np.int32)
    up.close()
    dp.close()
    store.compact(0.0, buckets=[3])
    return store, raws


def test_every_kind_of_extent_moves_and_nothing_changes(gpu_api):
    store, raws = mixed_store(gpu_api)
    plans = [capi.Plan(gpu_api, q.desc()) for q in QUERIES]
    proj = capi.Plan(gpu_api, _projection())
    try:
        want = [kc.evaluate(q, raws) for q in QUERIES]
        before_paths = []
        for q, p, w in zip(QUERIES, plans, want):
            kc.assert_rows_exact(_run(p, q, store), w, q, "before")
            before_paths.append(_paths(p))
        rows_before = _rows(proj, store)
        assert rows_before
        snap = _snapshot(store)
        live, _ = store.extent_bytes()
        assert live > 0
        _, slab_bytes = store.memory_info()
        res = store.reclaim(1.0)
        tm = capi.last_reclaim_timing(gpu_api)
        print(res, tm)
        assert res["bytes_freed"] == slab_bytes and res["slabs_deferred"] == 0   # every slab that existed before
        assert res["bytes_moved"] == live
        assert tm["rounds"] >= 1 and tm["copy_ms"] > 0
        assert store.extent_bytes() == (live, 0)
        assert _snapshot(store) == snap
        for q, p, w, paths in zip(QUERIES, plans, want, before_paths):
            kc.assert_rows_exact(_run(p, q, store), w, q, "after, same handle")
            assert _paths(p) == paths
            fresh = capi.Plan(gpu_api, q.desc())
            kc.assert_rows_exact(_run(fresh, q, store), w, q, "after, fresh handle")
            assert _paths(fresh) == paths
            fresh.close()
        assert _rows(proj, store) == rows_before
        fresh = capi.Plan(gpu_api, _projection())
        assert _rows(fresh, store) == rows_before
        fresh.close()
    finally:
        for p in plans + [proj]:
            p.close()
        store.close()


def _lineitem_table(api, monkeypatch, slab_mb):
    monkeypatch.setenv("SD_TUNE_STORE_SLAB_MB", str(slab_mb))
    return Table(api)


def test_dead_slabs_are_freed_without_copying(gpu_api, monkeypatch):
    t = _lineitem_table(gpu_api, monkeypatch, 2)
    store = t.store
    dp = capi.Plan(gpu_api, _lineitem_delete())
    dp.delete_store(store, [4.0])
    for i in range(NB):
        t.live[i] &= ~(t.cur[i][L_QUANTITY] < 4.0)
    dp.close()
    res = store.compact(0.0)
    assert res["batches_rewritten"] == NB
    _, slabs_before = store.memory_info()
    r = store.reclaim(0.0)
    print(r, capi.last_reclaim_timing(gpu_api))
    assert r["bytes_moved"] == 0 and r["slabs_freed"] >= 1 and r["slabs_deferred"] == 0
    _, slabs_after = store.memory_info()
    assert slabs_before - slabs_after == r["bytes_freed"]
    ref = capi.Store(gpu_api, lineitem.LINEITEM_SCHEMA)   # the same live rows encoded fresh
    for i in range(NB):
        ref.encode_batch(int(t.live[i].sum()), {c: (t.live_values(i, c), None) for c in RESIDENT}, t.m.batches[i].bucket_id,
                         t.m.batches[i].batch_id)
    _, fresh_slabs = ref.memory_info()
    assert slabs_after <= fresh_slabs + (2 << 20)
    q6 = capi.Plan(gpu_api, P.q6_plan())
    (got,), = _q(q6, store, P.Q6_LITERALS)
    assert got == pytest.approx(t.q6(), rel=1e-6)
    q6.close()
    ref.close()
    store.close()


def _lineitem_delete():
    b = PlanBuilder()
    q = b.col(T.DOUBLE, L_QUANTITY)
    b.filter(q < b.lit(T.DOUBLE))
    b.delete()
    return b.build()


def _oracle_check(api, store, t):
    """Q1 against the C oracle over the store's (compacted) bytes, Q6 against numpy."""
    from oracle import oracle
    q1 = capi.Plan(api, P.q1_plan())
    got = _q(q1, store, P.Q1_LITERALS)
    op = oracle.plan(P.q1_plan()).set_literals(P.Q1_LITERALS)
    for i in range(store.num_batches()):
        n, bucket, bid = store.batch_info(i)
        cols = [None] * 16
        for c in RESIDENT:
            cols[c] = store.get_buffer(i, c)
        op.submit(ColumnBatch(num_rows=n, columns=cols, batch_id=bid, bucket_id=bucket))
    assert_rowsets_match(got, op.finish(), 2)
    op.close()
    q1.close()
    q6 = capi.Plan(api, P.q6_plan())
    (v,), = _q(q6, store, P.Q6_LITERALS)
    assert v == pytest.approx(t.q6(), rel=1e-6)
    q6.close()


def test_memory_stays_bounded_over_cycles(gpu_api, monkeypatch):
    t = _lineitem_table(gpu_api, monkeypatch, 2)
    store = t.store
    store.compact(0.0)
    for i in range(NB):
        t.compacted(i)
    _, base = store.memory_info()
    bound = 3 * base + 4 * (2 << 20)
    for cycle in range(6):
        _statements(gpu_api, t)
        store.compact(0.0)
        for i in range(NB):
            t.compacted(i)
        r = store.reclaim(0.5)
        _, slabs = store.memory_info()
        print(cycle, r, slabs, bound)
        assert slabs <= bound, (cycle, slabs, bound)
        _oracle_check(gpu_api, store, t)
    store.close()


def test_an_open_scan_pins_its_memory(gpu_api):
    store, raws = mixed_store(gpu_api)
    q = kc.Query(["h"], [(AggFn.MIN, "s"), (AggFn.MAX, "s"), (AggFn.COUNT_STAR, None)])
    want = kc.evaluate(q, raws)
    plan = capi.Plan(gpu_api, q.desc())
    plan.reset().set_literals([])
    plan.scan_store(store)                        # scanned, not finished
    r1 = store.reclaim(1.0)
    assert r1["slabs_deferred"] >= 1 and r1["slabs_freed"] == 0 and r1["bytes_moved"] > 0
    assert store.extent_bytes()[1] > 0            # the replaced versions stay for the open scan
    plan._out_buf = capi.C.create_string_buffer(8)   # too small: SD_ERR_OVERFLOW first, then the repeat
    kc.assert_rows_exact(plan.finish(), want, q, "open scan")
    kc.assert_rows_exact(plan.finish(), want, q, "repeated finish")
    r2 = store.reclaim(0.0)
    assert r2["slabs_freed"] >= r1["slabs_deferred"] and r2["slabs_deferred"] == 0
    assert store.extent_bytes()[1] == 0
    kc.assert_rows_exact(_run(plan, q, store), want, q, "after")
    plan.close()
    # a plan destroyed after its store
    late = capi.Plan(gpu_api, q.desc())
    late.reset().set_literals([])
    late.scan_store(store)
    import torch
    torch.cuda.synchronize()   # the scan's kernels are done; its pin is still held
    store.close()
    late.close()


def test_reclaim_beside_queries_and_ingest(gpu_api):
    q = kc.Query(["k"], [(AggFn.COUNT_STAR, None), (AggFn.SUM, "i"), (AggFn.MIN, "s"), (AggFn.MAX, "d")])
    cases = [kc.make_batch(2049, "fast_nulls", seed=900 + i, groups=7, batch_id=i) for i in range(24)]
    store = capi.Store(gpu_api, STORE_SCHEMA)
    for b, _ in cases[:4]:
        store.put(b)
    prefix = {k: kc.evaluate(q, [c[1] for c in cases[:k]]) for k in range(4, len(cases) + 1)}
    errors, results, done = [], [], threading.Event()

    def ingest():
        try:
            for k in range(4, len(cases)):
                b, r = cases[k]
                if k % 2:
                    store.encode_batch(r.n, {c: (r.values[name], r.nulls.get(name)) for c, (name, _, _) in enumerate(kc.SCHEMA)},
                                       b.bucket_id, b.batch_id)
                else:
                    store.put(b)
        except Exception as e:   # pragma: no cover - reported below
            errors.append(e)
        finally:
            done.set()

    def query():
        p = capi.Plan(gpu_api, q.desc())
        try:
            while not done.is_set() or len(results) < 3:
                results.append(_run(p, q, store))
        except Exception as e:   # pragma: no cover
            errors.append(e)
        finally:
            p.close()

    th = [threading.Thread(target=ingest), threading.Thread(target=query)]
    for x in th:
        x.start()
    reclaims = 0
    while not done.is_set() or reclaims < 3:
        store.reclaim(1.0)
        reclaims += 1
    for x in th:
        x.join()
    assert not errors, errors
    for got in results:
        assert any(_same(got, w, q) for w in prefix.values()), got
    final = capi.Plan(gpu_api, q.desc())
    kc.assert_rows_exact(_run(final, q, store), prefix[len(cases)], q, "final")
    final.close()
    for i in range(store.num_batches()):
        _, _, bid = store.batch_info(i)
        if bid % 2 == 0 or bid < 4:
            b = cases[bid][0]
            for c in range(len(STORE_SCHEMA)):
                assert store.get_buffer(i, c) == bytes(b.columns[c]), (bid, c)
    store.reclaim(0.0)
    store.close()


def _same(got, want, q):
    try:
        kc.assert_rows_exact(got, want, q, "")
        return True
    except AssertionError:
        return False


def test_statements_after_a_reclaim(gpu_api, monkeypatch):
    t = _lineitem_table(gpu_api, monkeypatch, 2)
    store = t.store
    old = {(i, c): store.get_buffer(i, c) for i in range(NB) for c in RESIDENT}
    masks = [store.get_deletes(i) if t.m.mask[i] is not None else None for i in range(NB)]
    r = store.reclaim(1.0)
    assert r["bytes_moved"] > 0 and r["slabs_deferred"] == 0
    for i in range(NB):
        assert all(store.get_buffer(i, c) == old[(i, c)] for c in RESIDENT)
        for c in t.m.delta0[i]:
            assert store.get_delta(i, c, 0) == t.m.delta0[i][c]
        if masks[i] is not None:
            assert store.get_deletes(i) == masks[i]
    _statements(gpu_api, t)
    store.reclaim(1.0)
    pre = {(i, c): store.get_buffer(i, c) for i in range(NB) for c in RESIDENT}
    masked = [not t.live[i].all() or t.m.mask[i] is not None for i in range(NB)]
    store.compact(0.0)
    for i in range(NB):   # rewritten columns: the fixture writer's bytes of the live rows; the others as they were
        assert store.batch_info(i)[0] == int(t.live[i].sum())
        for c in RESIDENT:
            if t.dirty[i] and (masked[i] or c in t.delta_cols[i]):
                assert store.get_buffer(i, c) == encode_column(t.live_values(i, c), _typ(c)), (i, c)
            else:
                assert store.get_buffer(i, c) == pre[(i, c)], (i, c)
        t.compacted(i)
    store.reclaim(1.0)
    _oracle_check(gpu_api, store, t)
    store.close()


def test_compression_kept_and_refusals(gpu_api):
    store, _ = mixed_store(gpu_api)
    comp0, total0 = store.memory_info()
    store.reclaim(1.0)
    comp1, total1 = store.memory_info()
    assert total1 > 0 and comp0 * total1 == comp1 * total0   # the same compressible share
    before = (store.extent_bytes(), store.memory_info(), store.num_batches(), _snapshot(store))
    for f in (math.nan, -0.1, 1.5, -math.inf, math.inf):
        with pytest.raises(SdError) as e:
            store.reclaim(f)
        assert e.value.code == capi.SD_ERR_INVALID
    out = (capi.C.c_int64 * 4)()
    assert gpu_api.lib.sd_store_reclaim(None, 0.5, out) == capi.SD_ERR_INVALID
    assert (store.extent_bytes(), store.memory_info(), store.num_batches(), _snapshot(store)) == before
    store.close()


def test_reclaim_over_60m_rows(gpu_api):
    total, rpb, seed = 59_986_052, 200_000, 6
    store = capi.Store(gpu_api, lineitem.LINEITEM_SCHEMA)
    store.gen_lineitem(0, total, rpb, 128, seed, lineitem.Q1_COLUMN_MASK)
    b = PlanBuilder()
    ship = b.col(T.DATE, L_SHIPDATE)
    b.group_by(ship)
    b.count()
    hash_desc = b.build()
    q1, hp = capi.Plan(gpu_api, P.q1_plan()), capi.Plan(gpu_api, hash_desc)
    before = _q(q1, store, P.Q1_LITERALS)
    _, slabs = store.memory_info()
    r = store.reclaim(1.0)
    tm = capi.last_reclaim_timing(gpu_api)
    print(r, tm)
    assert tm["rounds"] >= 3 and r["bytes_freed"] == slabs and r["slabs_deferred"] == 0
    assert r["bytes_moved"] == store.extent_bytes()[0]
    after = _q(q1, store, P.Q1_LITERALS)
    assert_rowsets_match(after, before, 2)
    ships = np.concatenate([lineitem.lineitem_values(i * rpb, min(rpb, total - i * rpb), seed)["l_shipdate"]
                            for i in range((total + rpb - 1) // rpb)])
    u, n = np.unique(ships, return_counts=True)
    got = {r[0]: r[1] for r in _q(hp, store, [])}
    assert got == dict(zip(u.tolist(), n.tolist()))
    for p in (q1, hp):
        p.close()
    store.close()
