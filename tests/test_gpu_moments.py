"""STDDEV / VARIANCE / SKEWNESS / KURTOSIS on the device, in every group-table placement, against exact Fraction arithmetic
(tests/moments_reference.py) and Spark's row-order update.

Each test asserts through Plan.launch_log() that the engine took the placement it targets.  The data sets are the ones raw power
sums get wrong: mean 1e9 with sigma 1, sigma 1e-6 around 0, and groups whose magnitudes differ by many orders in one table."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import kernel_cases as kc
import moments_reference as R
from snappydata_b200 import capi
from snappydata_b200.capi import AggFn
from snappydata_b200.column_format import build_batch
from snappydata_b200.plan import PlanBuilder

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
FNS = R.MOMENT_FNS
STORE_SCHEMA = [(t, n) for _, t, n in kc.SCHEMA]


def moment_plan(keys, filter_lit=False):
    """keys ++ [COUNT(*), the six functions of d]; filter `i IS NULL OR i > lit` when asked"""
    b = PlanBuilder()
    e = {name: b.col(kc.TYPE[name], kc.COL[name], kc.NULLABLE[name]) for name in ["d", "i"] + list(keys)}
    if filter_lit:
        b.filter(e["i"].is_null() | (e["i"] > b.lit(kc.T.INT)))
    if keys:
        b.group_by(*[e[k] for k in keys])
    b.count()
    for fn in FNS:
        b.agg(fn, e["d"])
    return b.build()


def profile_values(profile, g, rng):
    """x per row of group g"""
    n = len(g)
    if profile == "big_mean":
        return 1e9 + rng.standard_normal(n)
    if profile == "tiny":
        return 1e-6 * rng.standard_normal(n)
    scale = 10.0 ** ((g % 7) - 2)                          # groups of very different magnitudes in one table
    return 10.0 ** ((g % 5) * 2) + scale * rng.standard_normal(n) * (1 + (g % 3))


def numeric_batch(n, kind, seed, groups, profile, batch_id=0, group_base=0, distinct_groups=False):
    """kernel_cases.make_batch with column d replaced by the profile's values (NULL masks kept)"""
    _, raw = kc.make_batch(n, kind, seed, groups, batch_id=batch_id, group_base=group_base, distinct_groups=distinct_groups)
    assert not raw.deltas and not len(raw.deletes)
    rng = np.random.default_rng(seed + 7)
    gid = np.array([int(k[1:]) if k[:1] == b"g" else int(k[3:]) for k in raw.values["k"]])
    raw.values["d"] = profile_values(profile, gid, rng)
    batch = build_batch(n, kc.SCHEMA, raw.values, raw.nulls, batch_id=batch_id, bucket_id=batch_id % 4, encoders=kc.ENCODERS[kind])
    batch.stats = None
    return batch, raw


def expected(keys, raws, lit=None):
    """{key tuple: [values of d]} over the live rows that pass the filter"""
    groups = {}
    for raw in raws:
        live = raw.live()
        cols = {name: raw.effective(name) for name in ["d", "i"] + list(keys)}
        for r in range(raw.n):
            if not live[r]:
                continue
            if lit is not None and not (cols["i"][1][r] or cols["i"][0][r] > lit):
                continue
            key = tuple(None if cols[k][1][r] else cols[k][0][r] for k in keys)
            groups.setdefault(key, []).append(None if cols["d"][1][r] else float(cols["d"][0][r]))
    return groups


def check(plan, desc, keys, raws, raw_partials, lit=None, what=""):
    """final rows of the device's partial rows against exact arithmetic and against Spark's row-order update"""
    want = expected(keys, raws, lit)
    got = plan.final_merge(raw_partials)
    nk = len(keys)
    assert sorted(repr(tuple(r[:nk])) for r in got) == sorted(repr(k) for k in want), what
    worst = 0.0
    for row in got:
        xs = want[tuple(row[:nk])]
        assert row[nk] == len(xs), what
        for fn, v in zip(FNS, row[nk + 1:]):
            ex = R.exact(fn, xs)
            assert R.close(fn, v, ex), (what, row[:nk], fn, v, ex)
            sp = R.evaluate(fn, R.welford(xs, R.ORDER[fn]))   # Spark's own row-order update agrees, to its own rounding
            assert (sp is None and v is None) or (math.isnan(sp) and math.isnan(v)) or abs(sp - v) <= max(1e-4 * abs(sp), 1e-4), \
                (what, fn, v, sp)
            if ex is not None and not math.isnan(ex) and ex != 0:
                worst = max(worst, abs(v - ex) / abs(ex))
    print(what, len(got), "groups, worst relative error", worst)
    return want


def run(plan, desc, batches, lits=(), store=None):
    plan.reset().set_literals(list(lits))
    if store is not None:
        plan.scan_store(store)
    else:
        for b in batches:
            plan.submit(b)
    return plan.finish_raw()


# accumulator -> (keys, groups drawn)
PLACEMENTS = {"nokey": ([], 8), "private": (["k"], 3), "shared_atomic": (["k"], 40), "global_atomic": (["k"], 1500),
              "hash": (["h"], 1500)}


@pytest.mark.parametrize("profile", ["big_mean", "tiny", "mixed"])
@pytest.mark.parametrize("accumulator", list(PLACEMENTS))
def test_placements_against_exact_arithmetic(gpu_api, monkeypatch, accumulator, profile):
    monkeypatch.setenv("SD_TUNE_CHUNK_ROWS", "2048")
    keys, groups = PLACEMENTS[accumulator]
    cases = [numeric_batch(n, kind, seed=300 + 10 * i + j, groups=groups, profile=profile, batch_id=2 * i + j)
             for i, n in enumerate((2049, 3 * 2048 + 77, 30000)) for j, kind in enumerate(("all_fast", "fast_nulls"))]
    batches, raws = [c[0] for c in cases], [c[1] for c in cases]
    desc = moment_plan(keys, filter_lit=True)
    plan = capi.Plan(gpu_api, desc)
    st = capi.Store(gpu_api, STORE_SCHEMA)
    try:
        for b in batches:
            st.put(b)
        for lit in (-900, 200):   # one cached plan, new literals
            for where, store in (("submit", None), ("store", st)):
                raw = run(plan, desc, batches, [lit], store)
                log = plan.launch_log()
                assert log and all(r["accumulator"] == accumulator for r in log), log
                want = check(plan, desc, keys, raws, raw, lit, f"{accumulator}/{profile}/{where}/{lit}")
        if profile == "big_mean":   # float64 sum x^2 of the same data misses the bar: the bar has teeth
            misses = [R.naive(AggFn.VAR_SAMP, xs) for xs in want.values() if sum(x is not None for x in xs) > 100]
            exact = [R.exact(AggFn.VAR_SAMP, xs) for xs in want.values() if sum(x is not None for x in xs) > 100]
            assert any(abs(a - b) > 1e-3 * abs(b) for a, b in zip(misses, exact))
    finally:
        st.close()
        plan.close()


@pytest.mark.parametrize("kind", ["fast_overlay", "rle", "fast_nulls"])
def test_deltas_deletes_nulls_nan_and_infinity(gpu_api, monkeypatch, kind):
    """kernel_cases batches: update deltas and delete masks (overlay and per-row paths), NULL runs, all-NULL groups, and groups
    holding NaN / +-inf (their results are NaN)."""
    monkeypatch.setenv("SD_TUNE_CHUNK_ROWS", "2048")
    cases = [kc.make_batch(n, kind, seed=40 + i, groups=9, batch_id=i) for i, n in enumerate(kc.BOUNDARY_SIZES)]
    for keys in ([], ["k"], ["h"]):
        desc = moment_plan(keys)
        plan = capi.Plan(gpu_api, desc)
        try:
            raw = run(plan, desc, [c[0] for c in cases])
            want = check(plan, desc, keys, [c[1] for c in cases], raw, None, f"{kind}/{keys}")
            if keys == ["k"]:
                assert any(any(x is not None and math.isnan(x) for x in xs) for xs in want.values())
        finally:
            plan.close()


def growth_batches():
    spec = [(100000, dict(groups=2)), (100000, dict(groups=100)), (100000, dict(groups=3000)),   # > 1 MB each: one launch each
            (75000, dict(groups=1, group_base=3000, distinct_groups=True))]
    return [numeric_batch(n, "fast_nulls", seed=777 + i, batch_id=i, profile="mixed", **kw) for i, (n, kw) in enumerate(spec)]


def test_placement_changes_hash_switch_and_grow(gpu_api, monkeypatch):
    """One execution of four launches: private -> shared-atomic -> global-atomic (the dense table re-indexed with its K words),
    then the switch to the hash table replays the earlier launches and the hash table grows and replays all four: the K words
    are rebuilt with each table."""
    monkeypatch.setenv("SD_TUNE_FLUSH_MB", "1")
    cases = growth_batches()
    desc = moment_plan(["k"])
    plan = capi.Plan(gpu_api, desc)
    try:
        raw = run(plan, desc, [c[0] for c in cases[:3]])
        assert [r["accumulator"] for r in plan.launch_log()] == ["private", "shared_atomic", "global_atomic"]
        check(plan, desc, ["k"], [c[1] for c in cases[:3]], raw, None, "growth dense")
        raw = run(plan, desc, [c[0] for c in cases])
        seq = [(r["accumulator"], r["replay"]) for r in plan.launch_log()]
        assert seq[:3] == [("private", None), ("shared_atomic", None), ("global_atomic", None)], seq
        assert seq[3:7] == [("hash", "hash_switch")] * 3 + [("hash", None)], seq
        assert seq[7:] and all(s == ("hash", "hash_grow") for s in seq[7:]), seq
        check(plan, desc, ["k"], [c[1] for c in cases], raw, None, "growth hash")
    finally:
        plan.close()


def test_no_rows_and_dense_partials_refused(gpu_api):
    desc = moment_plan([], filter_lit=True)
    plan = capi.Plan(gpu_api, desc)
    try:
        b, _ = numeric_batch(5000, "all_fast", seed=3, groups=4, profile="tiny")
        raw = run(plan, desc, [b], [10 ** 6])                      # every row filtered out
        assert capi.parse_row_stream(raw, desc.partial_schema()) == [[0] + [0.0] * 21]
        assert plan.final_merge(raw) == [[0] + [None] * 6]
        # the dense partials export / import: shifted sums of different GPUs do not add
        import ctypes as C
        import torch
        lib, buf = gpu_api.lib, torch.zeros(4096, dtype=torch.float64, device="cuda")
        assert lib.sd_plan_partials_layout(plan.h, None, None, None) == capi.SD_ERR_UNSUPPORTED
        assert lib.sd_plan_export_partials(plan.h, C.c_void_p(buf.data_ptr()), C.c_int64(buf.numel() * 8)) == capi.SD_ERR_UNSUPPORTED
        assert lib.sd_plan_import_partials(plan.h, C.c_void_p(buf.data_ptr()), C.c_int64(22 * 8)) == capi.SD_ERR_UNSUPPORTED
        assert plan.final_merge(plan.finish_raw()) == [[0] + [None] * 6]   # the refusals changed nothing
    finally:
        plan.close()


def test_exchange_on_two_gpus_equals_one_gpu():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29541", os.path.join(HERE, "moments_multirank_worker.py")], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "MOMENTS MULTIRANK OK" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])
