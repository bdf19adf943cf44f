"""The staged-only kernel lays its ring out by the widths a launch streams, and dense group-bys whose private table, image
tables and two such stages fit half an SM run two CTAs per SM.  A different grid only changes the order in which a group's
rows are summed: counts and exact sums stay identical, DOUBLE sums of generated lineitem agree to 1e-12 relative."""
import copy

import numpy as np
import pytest
import torch

from snappydata_b200 import capi, plan as P
from snappydata_b200.capi import AggFn
from snappydata_b200.column_format import compress_lz4

import kernel_cases as kc
from test_gpu_kernel_paths import STORE_SCHEMA, run_store
from test_gpu_scan_images import _Q, lineitem_store

pytestmark = pytest.mark.gpu

SHAPES = {"default": {}, "one_cta": {"SD_TUNE_GROUP_CTAS": "1"}, "verbatim": {"SD_TUNE_RING_LAYOUT": "verbatim"}}


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def scan_shape(gpu_api, monkeypatch, q, store, shape):
    """(partial rows, raw, launch log) of one execution under one of SHAPES, on a fresh plan."""
    for name in ("SD_TUNE_GROUP_CTAS", "SD_TUNE_RING_LAYOUT"):
        monkeypatch.delenv(name, raising=False)
    for name, value in SHAPES[shape].items():
        monkeypatch.setenv(name, value)
    plan = capi.Plan(gpu_api, q.desc())
    try:
        rows, raw = run_store(plan, q, store)
        return rows, raw, plan.launch_log()
    finally:
        plan.close()
        for name in SHAPES[shape]:
            monkeypatch.delenv(name, raising=False)


def assert_close_rows(a, b, what):
    """Same groups in the same order, integers identical, floating-point values within 1e-12 relative."""
    assert len(a) == len(b), what
    for ra, rb in zip(a, b):
        assert len(ra) == len(rb), what
        for x, y in zip(ra, rb):
            if isinstance(x, float) and isinstance(y, float):
                assert x == y or abs(x - y) <= 1e-12 * max(abs(x), abs(y)), (what, ra, rb)
            else:
                assert x == y, (what, ra, rb)


def test_q1_runs_two_ctas_per_sm_from_images(gpu_api, monkeypatch):
    """Q1 over device-generated lineitem: 15 B/row streamed, two CTAs per SM with a ring of >= 2 compact stages; one CTA
    (forced) and the verbatim layout give the same counts and sums to 1e-12."""
    q = _Q(P.q1_plan(), P.Q1_LITERALS)
    rows = 4_000_000
    st = lineitem_store(gpu_api, rows)
    try:
        got = {s: scan_shape(gpu_api, monkeypatch, q, st, s) for s in SHAPES}
        (log,) = got["default"][2]
        assert log["accumulator"] == "private" and log["grid"] == 2 * num_sms() and log["nstages"] >= 2, log
        assert log["streamed_bytes"] == 15 * rows, log
        for s in ("one_cta", "verbatim"):
            (other,) = got[s][2]
            assert other["grid"] == num_sms() and other["accumulator"] == "private", (s, other)
            assert_close_rows(got["default"][0], got[s][0], "q1 default / " + s)
    finally:
        st.close()


SMALL_QUERY = kc.Query(["k"], [(AggFn.COUNT_STAR, None), (AggFn.SUM, "i"), (AggFn.SUM, "l"), (AggFn.SUM, "d"), (AggFn.MIN, "d"),
                               (AggFn.MAX, "d")])


def batch_of(n, seed, batch_id, groups, narrow=False, dtab=None, nulls=False):
    """A kernel_cases batch with chosen value ranges: `narrow` integers take 1-byte images (else 2), `dtab` distinct DOUBLE
    values take a dictionary image of that many entries (None: kernel_cases' doubles, too many for one); `nulls` makes it
    a fast_nulls batch (its nullable columns stream verbatim)."""
    kind = "fast_nulls" if nulls else "all_fast"
    _, raw = kc.make_batch(n, kind, seed=seed, groups=groups, batch_id=batch_id)
    rng = np.random.default_rng(seed + 1)
    if narrow:
        raw.values["i"] = rng.integers(0, 200, n).astype(np.int32)
        raw.values["l"] = (kc.LONG_BASE + rng.integers(0, 200, n)).astype(np.int64)
    if dtab is not None:
        raw.values["d"] = (np.arange(dtab, dtype=np.float64) / 4.0 - 7.0)[np.arange(n) % dtab]
    b = kc.build_batch(n, kc.SCHEMA, raw.values, raw.nulls, batch_id=batch_id, bucket_id=batch_id % 4, encoders=kc.ENCODERS[kind])
    b.stats = None
    return b, raw


def lz4(b):
    c = copy.copy(b)
    c.columns = [None if x is None else compress_lz4(x, force=True) for x in b.columns]
    return c


ALL_SORTS = ("narrow_1entry", "wide_256entry", "lz4", "nulls")


def mixed_cases(groups, big_rows, sorts=ALL_SORTS):
    """BOUNDARY_SIZES batches of each sort, and one large batch so that the grid shows the CTAs per SM."""
    cases, bid = [], 0
    for sort in sorts:
        for n in kc.BOUNDARY_SIZES:
            if sort == "narrow_1entry":
                b, raw = batch_of(n, 100 + bid, bid, groups, narrow=True, dtab=1)
            elif sort == "wide_256entry":
                b, raw = batch_of(n, 100 + bid, bid, groups, dtab=256)
            elif sort == "lz4":
                b, raw = batch_of(n, 100 + bid, bid, groups, narrow=True, dtab=3)
                b = lz4(b)
            else:
                b, raw = batch_of(n, 100 + bid, bid, groups, nulls=True)
            cases.append((b, raw))
            bid += 1
    cases.append(batch_of(big_rows, 999, bid, groups, narrow=True, dtab=1))
    return cases


@pytest.mark.parametrize("groups,ctas,sorts", [(2, 2, ALL_SORTS), (9, 1, ALL_SORTS), (2, 2, ("narrow_1entry", "wide_256entry"))],
                         ids=["small_table", "large_table", "images_only"])
def test_mixed_batches_exact_at_the_predicted_shape(gpu_api, monkeypatch, groups, ctas, sorts):
    """One execution over 1- and 2-byte images, batches without images (LZ4 puts), fast_nulls batches and 1- / 256-entry
    DOUBLE tables: rows exact against the evaluator with the default shape and with one CTA forced.  The private table of
    three groups (the NULL key is one) x 8 slots, 48 KB, fits two CTAs per SM beside two stages of the widest widths these
    batches stream (22 B/row); that of ten groups, 160 KB, does not, and that launch keeps one CTA per SM.  Without the LZ4
    and NULL batches the stage regions of the image columns are narrower than their verbatim widths (1- next to 2-byte
    images sized at 2)."""
    monkeypatch.setenv("SD_TUNE_CHUNK_ROWS", "2048")
    q = SMALL_QUERY
    cases = mixed_cases(groups, 600_000, sorts)
    st = capi.Store(gpu_api, STORE_SCHEMA)
    try:
        for b, _ in cases:
            st.put(b)
        info = st.image_info()
        assert info["images"] > 0 and info["mismatches"] == 0, info
        want = kc.evaluate(q, [c[1] for c in cases])
        for shape in ("default", "one_cta"):
            rows, _, log = scan_shape(gpu_api, monkeypatch, q, st, shape)
            kc.assert_rows_exact(rows, want, q, f"mixed/{shape}")
            (rec,) = log
            assert rec["accumulator"] == "private" and not rec["full_paths"] and rec["nstages"] >= 2, rec
            assert rec["paths"]["all_fast"] > 0 and (rec["paths"]["fast_nulls"] > 0) == ("nulls" in sorts), rec
            expect = ctas if shape == "default" else 1
            assert rec["chunks"] >= 2 * num_sms() and rec["grid"] == expect * num_sms(), (shape, rec)
    finally:
        st.close()
