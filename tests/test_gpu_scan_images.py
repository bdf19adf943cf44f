"""Scan images (narrow byte-aligned copies of resident NOT NULL columns, sd_image.cu) change what the staged loads read and
nothing else: every case runs with images on and with SD_TUNE_NO_SCAN_IMAGES=1, and the partial rows must be exact against
the evaluator of tests/kernel_cases.py and the same bytes -- doubles bit for bit -- wherever the answer does not depend on
the order in which rows meet (assert_same_result: with atomics, which of -0.0 / +0.0 wins a MIN / MAX tie does)."""
import numpy as np
import pytest

from snappydata_b200 import capi, lineitem, plan as P
from snappydata_b200.capi import AggFn

import kernel_cases as kc
from test_gpu_kernel_paths import BOUNDARY_QUERY, STORE_SCHEMA, assert_same_result, run_store

pytestmark = pytest.mark.gpu


def scan_both(gpu_api, monkeypatch, q, store):
    """(rows, raw, launch log) with images, then without; a fresh plan each so no cached descriptors carry over."""
    out = []
    for off in (False, True):
        if off:
            monkeypatch.setenv("SD_TUNE_NO_SCAN_IMAGES", "1")
        else:
            monkeypatch.delenv("SD_TUNE_NO_SCAN_IMAGES", raising=False)
        plan = capi.Plan(gpu_api, q.desc())
        try:
            rows, raw = run_store(plan, q, store)
            out.append((rows, raw, plan.launch_log()))
        finally:
            plan.close()
    monkeypatch.delenv("SD_TUNE_NO_SCAN_IMAGES", raising=False)
    return out


@pytest.mark.parametrize("kind", ["all_fast", "fast_nulls", "fast_overlay"])
def test_images_match_verbatim_on_every_staged_path(gpu_api, monkeypatch, kind):
    """The boundary batch sizes of test_gpu_kernel_paths (1 .. 20,000 rows; images from 1024 rows): INT, LONG and
    dictionary codes give 2- and 1-byte offsets.  The kernel variant with the per-row paths (overlay batches) reads the
    verbatim values."""
    monkeypatch.setenv("SD_TUNE_CHUNK_ROWS", "2048")
    q = BOUNDARY_QUERY
    cases = [kc.make_batch(n, kind, seed=40 + i, groups=9, batch_id=i) for i, n in enumerate(kc.BOUNDARY_SIZES)]
    st = capi.Store(gpu_api, STORE_SCHEMA)
    try:
        for b, _ in cases:
            st.put(b)
        info = st.image_info()
        assert info["images"] > 0 and info["mismatches"] == 0, info
        (on_rows, on_raw, on_log), (_, off_raw, off_log) = scan_both(gpu_api, monkeypatch, q, st)
        kc.assert_rows_exact(on_rows, kc.evaluate(q, [c[1] for c in cases]), q, kind + "/images")
        assert_same_result(on_raw, off_raw, q, on_log, kind + " images on / off")
        (on,), (off,) = on_log, off_log
        assert on["paths"][kc.KIND_PATH[kind]] == len(cases) and on["nstages"] >= 2, on
        if kind == "fast_overlay":
            assert on["full_paths"] and on["streamed_bytes"] == off["streamed_bytes"], (on, off)
        else:
            assert on["streamed_bytes"] < off["streamed_bytes"], (on, off)
        print(kind, info, on["streamed_bytes"], off["streamed_bytes"])
    finally:
        st.close()


def special_batch(n, seed, batch_id):
    """A batch whose DOUBLE / FLOAT columns hold <= 256 distinct bit patterns: both zeros, two NaN payloads, +-inf."""
    _, raw = kc.make_batch(n, "all_fast", seed=seed, groups=5, batch_id=batch_id)
    rng = np.random.default_rng(seed)
    nan2 = np.frombuffer(np.uint64(0x7ff8000000000123).tobytes(), dtype=np.float64)[0]
    d = np.array([0.0, -0.0, np.nan, nan2, np.inf, -np.inf, 1.5, -2.25] + [x / 8 for x in range(240)], dtype=np.float64)
    raw.values["d"] = d[rng.integers(0, len(d), n)]
    f = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, 0.5], dtype=np.float32)
    raw.values["f"] = f[rng.integers(0, len(f), n)]
    batch = kc.build_batch(n, kc.SCHEMA, raw.values, raw.nulls, batch_id=batch_id, bucket_id=batch_id % 4, encoders=kc.ENCODERS["all_fast"])
    batch.stats = None
    return batch, raw


def test_dictionary_images_keep_zero_signs_and_nan_payloads(gpu_api, monkeypatch):
    q = kc.Query(["k"], [(AggFn.COUNT_STAR, None), (AggFn.SUM, "d"), (AggFn.MIN, "d"), (AggFn.MAX, "d"), (AggFn.SUM, "f"),
                        (AggFn.MIN, "f"), (AggFn.MAX, "f")])
    cases = [special_batch(n, 90 + i, i) for i, n in enumerate((1024, 4097, 20000))]
    st = capi.Store(gpu_api, STORE_SCHEMA)
    try:
        for b, _ in cases:
            st.put(b)
        info = st.image_info()
        assert info["mismatches"] == 0 and info["images"] >= 2 * len(cases), info
        (on_rows, on_raw, on_log), (_, off_raw, off_log) = scan_both(gpu_api, monkeypatch, q, st)
        kc.assert_rows_exact(on_rows, kc.evaluate(q, [c[1] for c in cases]), q, "special doubles")
        assert_same_result(on_raw, off_raw, q, on_log, "special doubles images on / off")
        assert sum(r["streamed_bytes"] for r in on_log) < sum(r["streamed_bytes"] for r in off_log)
    finally:
        st.close()


@pytest.mark.parametrize("accumulator", ["nokey", "private", "shared_atomic", "hash"])
def test_images_match_verbatim_in_every_placement(gpu_api, monkeypatch, accumulator):
    from test_gpu_kernel_paths import ACC_AGGS, ACC_SIZES, ACCUMULATORS
    monkeypatch.setenv("SD_TUNE_CHUNK_ROWS", "2048")
    keys, groups, base = ACCUMULATORS[accumulator]
    q = kc.Query(keys, ACC_AGGS)
    cases = [kc.make_batch(n, "all_fast", seed=700 + i, groups=groups, group_base=base, batch_id=i) for i, n in enumerate(ACC_SIZES + (200,))]
    st = capi.Store(gpu_api, STORE_SCHEMA)
    try:
        for b, _ in cases:
            st.put(b)
        (on_rows, on_raw, on_log), (_, off_raw, off_log) = scan_both(gpu_api, monkeypatch, q, st)
        kc.assert_rows_exact(on_rows, kc.evaluate(q, [c[1] for c in cases]), q, accumulator)
        assert_same_result(on_raw, off_raw, q, on_log, accumulator + " images on / off")
        assert all(r["accumulator"] == accumulator for r in on_log), on_log
        assert sum(r["streamed_bytes"] for r in on_log) < sum(r["streamed_bytes"] for r in off_log)
        assert st.image_info()["mismatches"] == 0
    finally:
        st.close()


def lineitem_store(gpu_api, rows, seed=3):
    st = capi.Store(gpu_api, lineitem.LINEITEM_SCHEMA)
    st.gen_lineitem(0, rows, 100_000, 8, seed, lineitem.Q1_COLUMN_MASK)
    return st


class _Q:   # Query-shaped wrapper around a PlanDesc for run_store
    def __init__(self, desc, lits):
        self._d, self._l = desc, lits

    def desc(self):
        return self._d

    def literals(self):
        return self._l


@pytest.mark.parametrize("query", ["q1", "q6"])
def test_generated_lineitem_streams_images(gpu_api, monkeypatch, query):
    """Device-generated lineitem: Q1 / Q6 give the same bytes with and without images, and read 15 / 12 bytes per row
    instead of 40 / 28 (l_extendedprice stays 8 bytes; quantity, discount, tax, flags 1 byte; shipdate 2)."""
    q = _Q(P.q1_plan(), P.Q1_LITERALS) if query == "q1" else _Q(P.q6_plan(), P.Q6_LITERALS)
    rows = 1_000_000
    st = lineitem_store(gpu_api, rows)
    try:
        info = st.image_info()
        assert info["images"] == 6 * 10 and info["mismatches"] == 0, info
        (_, on_raw, on_log), (_, off_raw, off_log) = scan_both(gpu_api, monkeypatch, q, st)
        assert on_raw == off_raw
        on_b, off_b = sum(r["streamed_bytes"] for r in on_log), sum(r["streamed_bytes"] for r in off_log)
        assert (on_b, off_b) == ((15 * rows, 40 * rows) if query == "q1" else (12 * rows, 28 * rows)), (on_b, off_b)
    finally:
        st.close()


def test_images_survive_update_delete_compact_and_reclaim(gpu_api, monkeypatch):
    """UPDATE / DELETE on an imaged store (the overlay path reads the verbatim values and keeps the images), then
    compaction (the rewritten columns get new images, so the scan streams them again) and reclaim (images move with their
    version): the same bytes with and without images, and no image fails its verification."""
    from snappydata_b200.column_format import SqlType as T
    from test_gpu_mutations import _update_plan
    from snappydata_b200.plan import L_DISCOUNT, L_QUANTITY, L_SHIPDATE
    q = _Q(P.q1_plan(), P.Q1_LITERALS)
    st = lineitem_store(gpu_api, 300_000, seed=11)
    up = capi.Plan(gpu_api, _update_plan(lambda b, c: {L_DISCOUNT: c[L_DISCOUNT] + b.lit(T.DOUBLE), L_QUANTITY: b.lit(T.DOUBLE)},
                                          lambda b, c: (c[L_SHIPDATE] >= b.lit(T.DATE)) & (c[L_SHIPDATE] <= b.lit(T.DATE))))
    dp = capi.Plan(gpu_api, _update_plan(None, lambda b, c: c[L_QUANTITY] < b.lit(T.DOUBLE)))
    try:
        assert up.update_store(st, [8800, 9000, 0.01, 7.0]) > 0
        assert dp.delete_store(st, [9.0]) > 0
        steps = [("mutated", None), ("compacted", lambda: st.compact(0.0)), ("reclaimed", lambda: st.reclaim(1.0))]
        for what, act in steps:
            if act:
                act()
            (_, on_raw, on_log), (_, off_raw, _) = scan_both(gpu_api, monkeypatch, q, st)
            assert on_raw == off_raw, what
            info = st.image_info()
            assert info["images"] > 0 and info["mismatches"] == 0, (what, info)
            paths = {k: sum(r["paths"][k] for r in on_log) for k in on_log[0]["paths"]}
            print(what, info, paths)
            if what == "mutated":
                assert paths["fast_overlay"] > 0, paths
            else:
                assert paths["fast_overlay"] == 0 and sum(r["streamed_bytes"] for r in on_log) < 40 * 300_000, (paths, on_log)
    finally:
        up.close()
        dp.close()
        st.close()
