"""Every code path the scan kernel picks, checked exactly against the evaluator of tests/kernel_cases.py.

The host chooses per batch between four decode paths, per plan between kernel shapes (rows per thread, ring or direct
loads) and per launch between group-table placements; within one execution the placement can change (dictionaries
grow: the dense table is re-indexed; past 65,536 groups the plan becomes its hash-table variant and replays).  Each test
asserts through Plan.launch_log() that the engine took the path it targets -- a heuristic change that moves it elsewhere
fails the test instead of silently covering less -- and compares every output row with the exact reference: counts,
integers, DECIMAL and strings equal, doubles bit for bit, NaN as NaN, MIN / MAX of +-0.0 as values.
"""
import math

import pytest

from snappydata_b200 import capi
from snappydata_b200.capi import AggFn

import kernel_cases as kc

pytestmark = pytest.mark.gpu

CHUNK = 2048
STORE_SCHEMA = [(t, n) for _, t, n in kc.SCHEMA]


def chunks(sizes, chunk_rows):
    return sum((n + chunk_rows - 1) // chunk_rows for n in sizes)


def launches(plan, replay=False):
    """The launch records of the plan's current execution (replays only when asked)."""
    return [r for r in plan.launch_log() if replay or r["replay"] is None]


def run_submit(plan, q, batches):
    plan.reset().set_literals(q.literals())
    for b in batches:
        plan.submit(b)
    raw = plan.finish_raw()
    return capi.parse_row_stream(raw, q.desc().partial_schema()), raw


def run_store(plan, q, store):
    plan.reset().set_literals(q.literals())
    plan.scan_store(store)
    raw = plan.finish_raw()
    return capi.parse_row_stream(raw, q.desc().partial_schema()), raw


def records(raw: bytes):
    out, pos = [], 0
    while pos < len(raw):
        n = int.from_bytes(raw[pos:pos + 8], "little")
        out.append(raw[pos:pos + 8 + n])
        pos += 8 + n
    return out


def assert_same_result(a: bytes, b: bytes, q, log, what):
    """A re-execution gives the same partial rows: byte for byte wherever the answer does not depend on the order in
    which rows meet -- the bits of a NaN (which NaN operand an addition propagates) and which of -0.0 / +0.0 wins a
    MIN / MAX tie do -- and, off the hash table (whose order depends on which of two colliding keys came first), in the
    same group order."""
    schema = q.desc().partial_schema()
    ra, rb = capi.parse_row_stream(a, schema), capi.parse_row_stream(b, schema)
    kc.assert_rows_exact(rb, ra, q, what + " (re-execution)")
    if not any(r["accumulator"] == "hash" for r in log):
        nk = len(q.keys)
        assert [r[:nk] for r in ra] == [r[:nk] for r in rb], what + ": re-execution changed the group order"
    same = sum(x == y for x, y in zip(sorted(records(a)), sorted(records(b))))
    print(f"{what}: {same} of {len(ra)} rows byte-identical on re-execution")


def new_store(gpu_api, batches):
    st = capi.Store(gpu_api, STORE_SCHEMA)
    for b in batches:
        st.put(b)
    return st


def check_both_paths(gpu_api, plan, q, batches, raws, what):
    """Submit path and resident store: exact against the evaluator; a second execution gives the same bytes."""
    want = kc.evaluate(q, raws)
    got, raw1 = run_submit(plan, q, batches)
    kc.assert_rows_exact(got, want, q, what + "/submit")
    log_submit = plan.launch_log()
    _, raw2 = run_submit(plan, q, batches)
    assert_same_result(raw1, raw2, q, log_submit, what + "/submit")
    st = new_store(gpu_api, batches)
    try:
        got, raw3 = run_store(plan, q, st)
        kc.assert_rows_exact(got, want, q, what + "/store")
        log_store = plan.launch_log()
        _, raw4 = run_store(plan, q, st)
        assert_same_result(raw3, raw4, q, log_store, what + "/store")
    finally:
        st.close()
    return log_submit, log_store


# ---- 1. every decode path at tile and work-item boundaries ----------------------------------------------------------
BOUNDARY_QUERY = kc.Query(["k"], kc.EVERY_AGG, filter_lit=-900)


@pytest.mark.parametrize("chunk_rows", [CHUNK, None], ids=["chunk2048", "default_chunk"])
def test_every_batch_path_at_tile_and_chunk_boundaries(gpu_api, monkeypatch, chunk_rows):
    """Batches of 1 .. 20,000 rows, mixed in one execution, on each of the four decode paths -- the general path once per
    encoding (RunLength, Dictionary, BigDictionary, BooleanBitSet) with NULL runs, update deltas (depth 0, depth 1, both,
    to NULL) and deletes on rows 0, 1023 / 1024 and the work-item edges, a deleted work item and an all-NULL tile."""
    if chunk_rows:
        monkeypatch.setenv("SD_TUNE_CHUNK_ROWS", str(chunk_rows))
    q = BOUNDARY_QUERY
    plan = capi.Plan(gpu_api, q.desc())
    try:
        expect_chunk = chunk_rows or 16384     # dense group plans default to two 8192-row chunks per work item
        for ki, kind in enumerate(kc.KINDS):
            cases = [kc.make_batch(n, kind, seed=100 * ki + i, groups=9, batch_id=i) for i, n in enumerate(kc.BOUNDARY_SIZES)]
            batches, raws = [c[0] for c in cases], [c[1] for c in cases]
            logs = check_both_paths(gpu_api, plan, q, batches, raws, kind)
            for log in logs:
                assert len(log) == 1, log
                (rec,) = log
                assert rec["paths"][kc.KIND_PATH[kind]] == len(batches), (kind, rec)
                assert sum(rec["paths"].values()) == len(batches), (kind, rec)
                assert rec["chunk_rows"] == expect_chunk and rec["chunks"] == chunks(kc.BOUNDARY_SIZES, expect_chunk), rec
                assert rec["full_paths"] == (kc.KIND_PATH[kind] in ("fast_overlay", "general")), rec
                assert rec["tile_rows"] == 1024 and rec["nstages"] >= 2, rec
                assert rec["accumulator"] == "shared_atomic", rec
                print(kind, "chunk", expect_chunk, rec)
    finally:
        plan.close()


# ---- 2. kernel shapes ------------------------------------------------------------------------------------------------
SHAPE_QUERY = kc.Query(["k"], [(AggFn.COUNT_STAR, None), (AggFn.SUM, "d"), (AggFn.SUM, "m"), (AggFn.AVG, "d"),
                               (AggFn.MIN, "d"), (AggFn.MAX, "i"), (AggFn.COUNT, "i")], filter_lit=-900)
SHAPE_SIZES = (1, 513, 1023, 1025, 2049, 3 * 2048 + 77, 20000)


@pytest.mark.parametrize("env,tile_rows,staged", [("SD_TUNE_RPT=2", 512, True), ("SD_TUNE_RPT=8", 2048, True),
                                                   ("SD_TUNE_STAGES=0", 1024, False)],
                         ids=["rpt2", "rpt8", "no_ring"])
def test_kernel_shapes_on_the_boundary_cases(gpu_api, monkeypatch, env, tile_rows, staged):
    name, value = env.split("=")
    monkeypatch.setenv(name, value)
    monkeypatch.setenv("SD_TUNE_CHUNK_ROWS", str(CHUNK))
    q = SHAPE_QUERY
    plan = capi.Plan(gpu_api, q.desc())
    try:
        for ki, kind in enumerate(("all_fast", "fast_nulls", "fast_overlay", "rle")):
            cases = [kc.make_batch(n, kind, seed=5000 + 100 * ki + i, groups=5, batch_id=i) for i, n in enumerate(SHAPE_SIZES)]
            logs = check_both_paths(gpu_api, plan, q, [c[0] for c in cases], [c[1] for c in cases], f"{env}/{kind}")
            for log in logs:
                (rec,) = log
                assert rec["tile_rows"] == tile_rows, rec
                assert (rec["nstages"] >= 2) if staged else (rec["nstages"] == 0), rec
                assert rec["paths"][kc.KIND_PATH[kind]] == len(SHAPE_SIZES), rec
                print(env, kind, rec)
    finally:
        plan.close()


# ---- 3. every accumulator with every slot operation -----------------------------------------------------------------
ACC_AGGS = [(AggFn.COUNT_STAR, None), (AggFn.COUNT, "i"), (AggFn.SUM, "i"), (AggFn.SUM, "l"), (AggFn.SUM, "f"),
            (AggFn.SUM, "d"), (AggFn.AVG, "m"), (AggFn.MIN, "d"), (AggFn.MAX, "d"), (AggFn.MIN, "f"), (AggFn.MAX, "f"),
            (AggFn.MIN, "s"), (AggFn.MAX, "s"), (AggFn.MIN, "i"), (AggFn.MAX, "m")]
ACC_SIZES = (2049, 3 * 2048 + 77, 20000)
# accumulator -> (keys, groups drawn, first group number)
ACCUMULATORS = {
    "nokey": ([], 8, 0),              # one group holding every special value
    "private": (["k"], 1, 1),         # the NaN group + the NULL key
    "shared_atomic": (["k"], 40, 0),
    "global_atomic": (["k"], 1500, 0),
    "hash": (["h"], 1500, 0),         # INT key: the hash-table plan
}


@pytest.mark.parametrize("accumulator", list(ACCUMULATORS))
def test_every_accumulator_with_every_slot_op(gpu_api, monkeypatch, accumulator):
    """COUNT(*), COUNT, SUM / AVG of INT, LONG (wrapping), FLOAT, DOUBLE, DECIMAL (carrying low halves), MIN / MAX of
    integers, doubles (NaN, +-inf, +-0.0, all-NULL groups) and strings (bytes >= 0x80, '', prefixes) in each placement."""
    monkeypatch.setenv("SD_TUNE_CHUNK_ROWS", str(CHUNK))
    keys, groups, base = ACCUMULATORS[accumulator]
    q = kc.Query(keys, ACC_AGGS)
    cases = [kc.make_batch(n, kind, seed=9000 + 10 * i + j, groups=groups, group_base=base, batch_id=i)
             for i, n in enumerate(ACC_SIZES) for j, kind in enumerate(("all_fast", "fast_nulls"))]
    plan = capi.Plan(gpu_api, q.desc())
    try:
        for log in check_both_paths(gpu_api, plan, q, [c[0] for c in cases], [c[1] for c in cases], accumulator):
            assert log and all(r["accumulator"] == accumulator for r in log), log
            print(accumulator, log)
    finally:
        plan.close()
    if accumulator == "nokey":        # the one group saw NaN and both infinities: SUM and MAX are NaN, MIN is -inf
        (row,) = kc.evaluate(q, [c[1] for c in cases])
        assert math.isnan(row[5]) and row[8] == -math.inf and math.isnan(row[9])


# ---- 4. placement changes within one execution ----------------------------------------------------------------------
GROWTH_QUERY = kc.Query(["k"], [(AggFn.COUNT_STAR, None), (AggFn.SUM, "d"), (AggFn.SUM, "m"), (AggFn.MIN, "d"),
                                (AggFn.MAX, "s")])


def growth_batches():
    """Key dictionaries that grow batch by batch: 3 groups (with NULL), ~100, ~3000, then ~69,000 new keys (> 65,536)."""
    spec = [(60000, dict(groups=2)), (60000, dict(groups=100)), (60000, dict(groups=3000)),
            (75000, dict(groups=1, group_base=3000, distinct_groups=True))]
    return [kc.make_batch(n, "fast_nulls", seed=777 + i, batch_id=i, **kw) for i, (n, kw) in enumerate(spec)]


def test_placement_changes_within_one_submit_execution(gpu_api, monkeypatch):
    """One execution, one launch per batch (flushed at 1 MB): private -> shared-atomic -> global-atomic (re-indexing the
    dense table each time), then the switch to the hash table replays the three earlier launches, and the hash table
    grows at the end and replays all four."""
    monkeypatch.setenv("SD_TUNE_FLUSH_MB", "1")
    q = GROWTH_QUERY
    cases = growth_batches()
    want = kc.evaluate(q, [c[1] for c in cases])
    plan = capi.Plan(gpu_api, q.desc())
    try:
        # the first three batches alone: the dense table is re-indexed twice and read back as it is
        got, _ = run_submit(plan, q, [c[0] for c in cases[:3]])
        kc.assert_rows_exact(got, kc.evaluate(q, [c[1] for c in cases[:3]]), q, "submit growth, dense")
        seq = [r["accumulator"] for r in plan.launch_log()]
        assert seq == ["private", "shared_atomic", "global_atomic"], seq
        # all four: past 65,536 groups the plan switches to the hash table
        got, raw1 = run_submit(plan, q, [c[0] for c in cases])
        kc.assert_rows_exact(got, want, q, "submit growth")
        log = plan.launch_log()
        print(log)
        seq = [(r["accumulator"], r["replay"]) for r in log]
        assert seq[:3] == [("private", None), ("shared_atomic", None), ("global_atomic", None)], seq
        assert seq[3:7] == [("hash", "hash_switch")] * 3 + [("hash", None)], seq
        grow = seq[7:]
        assert grow and len(grow) % 4 == 0 and all(s == ("hash", "hash_grow") for s in grow), seq
        _, raw2 = run_submit(plan, q, [c[0] for c in cases])
        assert_same_result(raw1, raw2, q, log, "submit growth")
    finally:
        plan.close()


def test_placement_changes_across_incremental_store_segments(gpu_api):
    """The same batches put into a resident store one by one, the cached query re-executed after each: the new batches
    become incremental scan segments, the dictionaries grow between executions, and the last one needs the hash table.
    Every segment must then be rebuilt for the hash kernel (regression: segments built for the dense table were launched
    by the hash kernel after the switch)."""
    q = GROWTH_QUERY
    cases = growth_batches()
    plan = capi.Plan(gpu_api, q.desc())
    st = capi.Store(gpu_api, STORE_SCHEMA)
    try:
        expect = ["private", "shared_atomic", "global_atomic", "hash"]
        for i, (b, _) in enumerate(cases):
            st.put(b)
            want = kc.evaluate(q, [c[1] for c in cases[: i + 1]])
            got, raw = run_store(plan, q, st)
            kc.assert_rows_exact(got, want, q, f"store growth {i}")
            log = plan.launch_log()
            print(i, log)
            first = launches(plan)
            assert first and all(r["accumulator"] == expect[i] for r in first), log
            if i == 3:
                assert any(r["replay"] == "hash_grow" for r in log), log
            _, raw2 = run_store(plan, q, st)
            assert_same_result(raw, raw2, q, log, f"store growth {i}")
    finally:
        st.close()
        plan.close()
