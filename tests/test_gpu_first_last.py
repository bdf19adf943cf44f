"""FIRST / LAST (with and without ignoreNulls) on the device, exact against the two restatements of Spark's rule in
tests/first_last_reference.py: the row-at-a-time update and the numpy first / last occurrence.

Each test pins through Plan.launch_log() the placement or path it targets.  Values pass through unchanged, so every field is
compared exactly: doubles by their bits (NaN payloads, -0.0), strings and DECIMAL(38, 2) by value."""
import struct

import numpy as np
import pytest

import first_last_reference as R
import kernel_cases as kc
from snappydata_b200 import capi
from snappydata_b200.capi import AggFn
from snappydata_b200.column_format import SqlType as T, build_batch, encode_delete, encode_delta, encode_wide_decimal, unsafe_row
from snappydata_b200.plan import PlanBuilder

pytestmark = pytest.mark.gpu

CHUNK = 2048
STORE_SCHEMA = [(t, n) for _, t, n in kc.SCHEMA]
# (k's update deltas hold strings its dictionary lacks: FIRST / LAST over it are refused, see the store test)
TYPED = ["i", "l", "f", "d", "m", "s", "b", "t", "sh", "dt"]
EVERY = [(AggFn.COUNT_STAR, None)] + [(fn, c) for c in TYPED for fn in R.ORDER_FNS]
# a plan small enough for the private per-thread tables
SMALL = [(AggFn.COUNT_STAR, None), (AggFn.FIRST, "d"), (AggFn.LAST, "d"), (AggFn.FIRST_IGNORE_NULLS, "s"),
         (AggFn.LAST_IGNORE_NULLS, "i"), (AggFn.FIRST, "m"), (AggFn.LAST_IGNORE_NULLS, "b")]


def rebuild(raw: kc.RawBatch, batch_id: int, kind: str = "fast_nulls"):
    """the ColumnBatch of a RawBatch whose base values a test has changed (deltas and delete mask as make_batch writes them)"""
    batch = build_batch(raw.n, kc.SCHEMA, raw.values, raw.nulls, batch_id=batch_id, bucket_id=batch_id % 4, encoders=kc.ENCODERS[kind])
    batch.stats = None
    for depth, name, pos, v, dn in raw.deltas:
        (batch.delta0 if depth == 0 else batch.delta1)[kc.COL[name]] = encode_delta(raw.n, pos, v, kc.TYPE[name], dn)
    if len(raw.deletes):
        batch.delete_mask = encode_delete(raw.n, raw.deletes)
    return batch


def run(plan, desc, batches=(), lits=(), store=None, rows=None):
    plan.reset().set_literals(list(lits))
    if rows is not None:
        plan.submit_rows(*rows)
    for b in batches:
        plan.submit(b)
    if store is not None:
        plan.scan_store(store)
    return capi.parse_row_stream(plan.finish_raw(), desc.partial_schema())


def check(got, keys, aggs, raws, lit=None, what=""):
    want = R.update_rows(keys, aggs, raws, lit)
    R.assert_rows_equal(got, want, len(keys), what + " vs row rule")
    R.assert_rows_equal(got, R.numpy_rows(keys, aggs, raws, lit), len(keys), what + " vs numpy")


def accumulators(plan):
    return [r["accumulator"] for r in plan.launch_log()]


ACCUMULATORS = {"nokey": ([], 1, 0), "private": (["k"], 1, 1), "shared_atomic": (["k"], 40, 0),
                "global_atomic": (["k"], 1500, 0), "hash": (["h"], 1500, 0)}


@pytest.mark.parametrize("accumulator", list(ACCUMULATORS))
def test_every_accumulator(gpu_api, monkeypatch, accumulator):
    """submit path and resident store, batches of the staged and the NULL-aware paths"""
    monkeypatch.setenv("SD_TUNE_CHUNK_ROWS", str(CHUNK))
    keys, groups, base = ACCUMULATORS[accumulator]
    cases = [kc.make_batch(n, kind, seed=6100 + 10 * i + j, groups=groups, group_base=base, batch_id=2 * i + j)
             for i, n in enumerate((3 * 2048 + 77, 20000)) for j, kind in enumerate(("all_fast", "fast_nulls"))]
    raws = [c[1] for c in cases]
    desc = R.desc(keys, SMALL)
    plan = capi.Plan(gpu_api, desc)
    st = capi.Store(gpu_api, STORE_SCHEMA)
    try:
        check(run(plan, desc, [c[0] for c in cases]), keys, SMALL, raws, what=accumulator + "/submit")
        assert accumulators(plan) and set(accumulators(plan)) == {accumulator}, plan.launch_log()
        for c in cases:
            st.put(c[0])
        check(run(plan, desc, store=st), keys, SMALL, raws, what=accumulator + "/store")
        assert set(accumulators(plan)) == {accumulator}, plan.launch_log()
    finally:
        st.close()
        plan.close()


@pytest.mark.parametrize("keys", [[], ["h"]], ids=["nokey", "hash"])
def test_every_type_and_batch_path_at_boundaries(gpu_api, monkeypatch, keys):
    """every kernel_cases kind (staged, NULL-aware, overlay and general paths; dictionary, RLE, bit-set and raw encodings) at the
    tile / work-item boundary sizes, 2048-row work items, and a filter that rejects the first chunks of every batch: the winning
    row is met by a CTA other than the first"""
    monkeypatch.setenv("SD_TUNE_CHUNK_ROWS", str(CHUNK))
    batches, raws = [], []
    for i, n in enumerate(kc.BOUNDARY_SIZES):
        kind = kc.KINDS[i % len(kc.KINDS)]
        _, raw = kc.make_batch(n, kind, seed=7300 + i, groups=6, batch_id=i)
        raw.values["i"][: (n * 3) // 4] = -1000        # base rows of the first three quarters fail `i > 0` (deltas may revive some)
        batches.append(rebuild(raw, i, kind))
        raws.append(raw)
    desc = R.desc(keys, EVERY, lit=0)
    plan = capi.Plan(gpu_api, desc)
    try:
        check(run(plan, desc, batches, [0]), keys, EVERY, raws, 0, "boundaries")
        paths = {k: sum(r["paths"][k] for r in plan.launch_log()) for k in ("all_fast", "fast_nulls", "fast_overlay", "general")}
        assert all(v > 0 for v in paths.values()), paths
    finally:
        plan.close()


def test_doubles_by_bits_and_wide_decimal_and_strings(gpu_api):
    """-0.0, +0.0 and NaNs of distinct payloads come back with their bits; DECIMAL(38, 2) and raw / dictionary STRINGs by value"""
    n = 5000
    rng = np.random.default_rng(3)
    sch = [("g", T.INT, False), ("x", T.DOUBLE, True), ("w", T.DECIMAL, True), ("s", T.STRING, True)]
    out = []
    for bi, enc in enumerate(("uncompressed", "dictionary")):
        x = rng.standard_normal(n)
        x[rng.random(n) < 0.3] = -0.0
        x[rng.random(n) < 0.2] = 0.0
        for j in np.flatnonzero(rng.random(n) < 0.3):
            x[j] = R.nan_with_payload(int(j) * 7919 + bi)
        g = rng.integers(0, 50, n).astype(np.int32)
        w = [int(v) * 10 ** 20 + int(u) for v, u in zip(rng.integers(-10 ** 15, 10 ** 15, n), rng.integers(0, 10 ** 18, n))]
        s = np.array([b"s%05d\x80" % int(v) for v in rng.integers(0, 300, n)], dtype=object)
        nulls = {"x": rng.random(n) < 0.1, "w": rng.random(n) < 0.1, "s": rng.random(n) < 0.1}
        data = {"g": g, "x": x, "w": np.array(w, dtype=object), "s": s}
        batch = build_batch(n, [c for c in sch if c[0] != "w"], data, nulls, batch_id=bi, encoders={"s": enc})
        batch.columns.insert(2, encode_wide_decimal(w, nulls["w"]))
        batch.stats = None
        out.append((batch, data, nulls))
    b = PlanBuilder()
    gc, xc = b.col(T.INT, 0, False), b.col(T.DOUBLE, 1, True)
    wc, sc = b.col(T.DECIMAL, 2, True, scale=2, precision=38), b.col(T.STRING, 3, True)
    b.group_by(gc)
    for fn in R.ORDER_FNS:
        b.agg(fn, xc).agg(fn, wc).agg(fn, sc)
    desc = b.build()
    plan = capi.Plan(gpu_api, desc)
    try:
        got = run(plan, desc, [o[0] for o in out])
    finally:
        plan.close()
    want = {}
    for _, data, nulls in out:   # row-at-a-time
        for r in range(n):
            key = int(data["g"][r])
            bufs = want.setdefault(key, [[None, False] for _ in range(12)])
            for a, fn in enumerate(R.ORDER_FNS):
                for c, col in enumerate(("x", "w", "s")):
                    v = None if nulls[col][r] else (float(data[col][r]) if col == "x" else data[col][r])
                    if R.ignores_nulls(fn) and v is None:
                        continue
                    buf = bufs[3 * a + c]
                    if R.is_last(fn) or not buf[1]:
                        buf[0] = v
                    buf[1] = True
    R.assert_rows_equal(got, [[k] + [f for b_ in v for f in b_] for k, v in want.items()], 1, "bits")
    assert any(R.is_nan(x) for r in got for x in r), "some winner is a NaN"


def test_row_buffer_then_batches_and_no_rows(gpu_api):
    """the row-buffer batch of sd_rows_submit is the first batch of the scan; no rows in: [NULL, false] without keys, no rows
    with keys"""
    aggs = [(AggFn.FIRST, "i"), (AggFn.LAST, "i"), (AggFn.FIRST_IGNORE_NULLS, "d"), (AggFn.LAST_IGNORE_NULLS, "s")]
    batch, raw = kc.make_batch(3000, "fast_nulls", seed=5, groups=3)
    desc = R.desc([], aggs)
    used = [n for n, _, _ in kc.SCHEMA if n in ("i", "d", "s")]
    rvals = [(7, None, b"row-first"), (None, 2.5, None), (8, None, b"")]
    rows = b""
    for v in rvals:
        u = unsafe_row([(kc.TYPE[c], x) for c, x in zip(used, v)])
        rows += struct.pack("<q", len(u)) + u
    rb = kc.RawBatch(3, {c: np.array([v[j] if v[j] is not None else (b"" if c == "s" else 0) for v in rvals],
                                      dtype=object if c == "s" else (np.float64 if c == "d" else np.int32))
                         for j, c in enumerate(used)},
                     {c: np.array([v[j] is None for v in rvals]) for j, c in enumerate(used)})
    plan = capi.Plan(gpu_api, desc)
    try:
        check(run(plan, desc, [batch], rows=(rows, 3)), [], aggs, [rb, raw], what="row buffer first")
        R.assert_rows_equal(run(plan, desc), [[None, False] * 4], 0, "no rows, no keys")
        kd = R.desc(["h"], aggs)
        kp = capi.Plan(gpu_api, kd)
        try:
            assert run(kp, kd) == []
        finally:
            kp.close()
    finally:
        plan.close()


def test_placement_changes_and_replays_in_one_execution(gpu_api, monkeypatch):
    """one launch per batch (flushed at 1 MB): private -> shared-atomic -> global-atomic, the switch to the hash table replays
    the three, the hash table grows and replays all four; the order keys are the same in every replay"""
    monkeypatch.setenv("SD_TUNE_FLUSH_MB", "1")
    spec = [(60000, dict(groups=2)), (60000, dict(groups=100)), (60000, dict(groups=3000)),
            (75000, dict(groups=1, group_base=3000, distinct_groups=True))]
    cases = [kc.make_batch(n, "fast_nulls", seed=8800 + i, batch_id=i, **kw) for i, (n, kw) in enumerate(spec)]
    aggs = [(AggFn.COUNT_STAR, None), (AggFn.FIRST, "d"), (AggFn.LAST, "s"), (AggFn.FIRST_IGNORE_NULLS, "i"), (AggFn.LAST_IGNORE_NULLS, "m")]
    desc = R.desc(["k"], aggs)
    plan = capi.Plan(gpu_api, desc)
    try:
        check(run(plan, desc, [c[0] for c in cases]), ["k"], aggs, [c[1] for c in cases], what="growth")
        seq = [(r["accumulator"], r["replay"]) for r in plan.launch_log()]
        first = [a for a, rp in seq if rp is None]
        assert len(first) == 4 and first[3] == "hash" and len(set(first[:3])) >= 2, seq
        assert set(first[:3]) <= {"private", "shared_atomic", "global_atomic"}, seq
        assert seq.count(("hash", "hash_switch")) == 3, seq
        assert ("hash", "hash_grow") in seq and seq[-1] == ("hash", "hash_grow"), seq
    finally:
        plan.close()


def _fold(raw: kc.RawBatch):
    """the batch's current values as base values (deltas folded in); the delete mask stays"""
    for c in list(raw.values):
        v, nl = raw.effective(c)
        raw.values[c] = np.array(v, dtype=raw.values[c].dtype)
        if c in raw.nulls:
            raw.nulls[c] = nl
    raw.deltas = []


def test_store_incremental_mutations_and_compaction(gpu_api):
    """resident store: an incremental re-scan after the store grows; then after a device UPDATE, a DELETE and a compaction
    that renumbers the ordinals"""
    cases = [kc.make_batch(n, kind, seed=9100 + i, groups=7, batch_id=i)
             for i, (n, kind) in enumerate(((5000, "fast_overlay"), (9000, "fast_nulls"), (4097, "all_fast")))]
    raws = [c[1] for c in cases]
    aggs = [(AggFn.FIRST, "l"), (AggFn.LAST, "l"), (AggFn.FIRST_IGNORE_NULLS, "d"), (AggFn.LAST, "s"), (AggFn.COUNT_STAR, None)]
    desc = R.desc(["k"], aggs)
    plan = capi.Plan(gpu_api, desc)
    st = capi.Store(gpu_api, STORE_SCHEMA)
    try:
        st.put(cases[0][0])
        st.put(cases[1][0])
        check(run(plan, desc, store=st), ["k"], aggs, raws[:2], what="store")
        st.put(cases[2][0])
        check(run(plan, desc, store=st), ["k"], aggs, raws, what="store grown")
        b = PlanBuilder()   # UPDATE SET l = 77 WHERE i > 900
        ic = b.col(T.INT, kc.COL["i"], True)
        b.filter(ic > b.lit(T.INT))
        b.update({kc.COL["l"]: b.lit(T.LONG)})
        up = capi.Plan(gpu_api, b.build())
        b = PlanBuilder()   # DELETE WHERE i < -900
        ic = b.col(T.INT, kc.COL["i"], True)
        b.filter(ic < b.lit(T.INT))
        b.delete()
        dp = capi.Plan(gpu_api, b.build())
        try:
            up.update_store(st, [900, 77])
            dp.delete_store(st, [-900])
        finally:
            up.close()
            dp.close()
        for raw in raws:
            _fold(raw)
            live = raw.live()
            i, inul = raw.values["i"], raw.nulls["i"]
            raw.values["l"] = np.where(live & ~inul & (i > 900), 77, raw.values["l"]).astype(np.int64)
            dels = np.flatnonzero(live & ~inul & (i < -900))
            raw.deletes = np.union1d(raw.deletes, dels).astype(np.int32)
        check(run(plan, desc, store=st), ["k"], aggs, raws, what="after UPDATE / DELETE")
        kd = R.desc(["h"], [(AggFn.LAST, "k")])   # k's deltas hold strings its dictionary lacks: refused until compacted
        kp = capi.Plan(gpu_api, kd)
        try:
            with pytest.raises(capi.SdError) as e:
                run(kp, kd, store=st)
            assert e.value.code == capi.SD_ERR_UNSUPPORTED, e.value
            st.compact(0.0)
            check(run(plan, desc, store=st), ["k"], aggs, raws, what="after compaction")
            check(run(kp, kd, store=st), ["h"], [(AggFn.LAST, "k")], raws, what="LAST(k) after compaction")
        finally:
            kp.close()
    finally:
        st.close()
        plan.close()


@pytest.mark.parametrize("shape", ["rollup", "cube"])
def test_grouping_sets_against_one_group_by_per_set(gpu_api, shape):
    # (no update deltas of k: a hash-table STRING key that exists only in a delta has no device record)
    cases = [kc.make_batch(n, kind, seed=9500 + i, groups=30, batch_id=i) for i, (n, kind) in enumerate(((7000, "fast_nulls"), (6000, "all_fast")))]
    raws = [c[1] for c in cases]
    aggs = [(AggFn.COUNT_STAR, None), (AggFn.FIRST, "d"), (AggFn.LAST_IGNORE_NULLS, "s"), (AggFn.LAST, "m")]
    b = PlanBuilder()
    e = {n: b.col(kc.TYPE[n], kc.COL[n], kc.NULLABLE[n], scale=kc.DEC_SCALE if kc.TYPE[n] == T.DECIMAL else 0) for n in ("k", "d", "s", "m", "sh")}
    (b.rollup if shape == "rollup" else b.cube)(e["k"], e["sh"])
    for fn, c in aggs:
        b.agg(fn, e[c] if c else None)
    desc = b.build()
    plan = capi.Plan(gpu_api, desc)
    try:
        got = run(plan, desc, [c[0] for c in cases])
    finally:
        plan.close()
    masks = [0, 1, 3] if shape == "rollup" else [0, 1, 2, 3]
    want = []
    for m in masks:
        present = [k for j, k in enumerate(("k", "sh")) if not (m >> (1 - j)) & 1]
        pdesc = R.desc(present, aggs)
        pp = capi.Plan(gpu_api, pdesc)
        try:
            plain = run(pp, pdesc, [c[0] for c in cases])
        finally:
            pp.close()
        R.assert_rows_equal(plain, R.update_rows(present, aggs, raws), len(present), f"plain set {m}")
        for r in plain:
            kv = dict(zip(present, r[: len(present)]))
            want.append([kv.get("k"), kv.get("sh"), m] + r[len(present):])
    R.assert_rows_equal(got, want, 3, shape)


def test_drop_duplicates_shaped_hash_group_by_60m_rows(gpu_api):
    """GROUP BY key with FIRST of four other columns over 60 M rows in 60 batches: every one of ~4 M groups against numpy"""
    n, nb, ng = 1_000_000, 60, 4_000_000
    sch = [("key", T.LONG, False), ("a", T.LONG, False), ("b", T.DOUBLE, False), ("c", T.INT, False), ("dt", T.DATE, False)]
    rng = np.random.default_rng(60)
    cols = {c: [] for c, _, _ in sch}
    b = PlanBuilder()
    e = [b.col(t, j, nl) for j, (_, t, nl) in enumerate(sch)]
    b.group_by(e[0])
    for x in e[1:]:
        b.first(x)
    desc = b.build()
    plan = capi.Plan(gpu_api, desc)
    try:
        plan.reset()
        for bi in range(nb):
            data = {"key": rng.integers(0, ng, n), "a": rng.integers(-10 ** 15, 10 ** 15, n), "b": rng.standard_normal(n),
                    "c": rng.integers(-2 ** 31, 2 ** 31, n).astype(np.int32), "dt": rng.integers(0, 20000, n).astype(np.int32)}
            batch = build_batch(n, sch, data, {}, batch_id=bi)
            batch.stats = None
            plan.submit(batch)
            for c in cols:
                cols[c].append(data[c])
        raw = plan.finish_raw()
        assert {r["accumulator"] for r in plan.launch_log()} == {"hash"}
    finally:
        plan.close()
    allc = {c: np.concatenate(v) for c, v in cols.items()}
    keys, first = np.unique(allc["key"], return_index=True)
    # partial rows: [int64 size][null bits (8)][key][a][b][c][dt][5 x 8 fields: values and valueSet flags]
    width = 8 + 8 * 9
    arr = np.frombuffer(raw, dtype=np.int64).reshape(-1, 1 + width // 8)
    assert (arr[:, 0] == width).all()
    assert (arr[:, 1] == 0).all()                                 # no NULL field
    order = np.argsort(arr[:, 2], kind="stable")
    got = arr[order]
    assert np.array_equal(got[:, 2], keys), "groups"
    assert np.array_equal(got[:, 3], allc["a"][first])
    assert np.array_equal(got[:, 5].view(np.float64).view(np.int64), allc["b"][first].view(np.int64))
    assert np.array_equal(got[:, 7].astype(np.int32), allc["c"][first])
    assert np.array_equal(got[:, 9].astype(np.int32), allc["dt"][first])
    assert (got[:, [4, 6, 8, 10]] & 0xff == 1).all()             # valueSet
