"""COVAR_POP / COVAR_SAMP / CORR on the device, in every group-table placement, against exact Fraction arithmetic
(tests/covariance_reference.py) and Spark's row-order update.

Each test asserts through Plan.launch_log() that the engine took the placement it targets.  The data sets are the ones raw sums
get wrong: x and y with mean 1e9 and sigma 1 (correlation about 0.9, 0 and exactly -1), sigma 1e-6 around 0, and groups whose
magnitudes differ by many orders in one table.  The plans carry COUNT(*), SUM(x) and STDDEV(x) beside the three functions."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import covariance_reference as R
import kernel_cases as kc
import moments_reference as MR
from snappydata_b200 import capi
from snappydata_b200.capi import AggFn
from snappydata_b200.column_format import SqlType as T, build_batch
from snappydata_b200.plan import PlanBuilder

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
FNS = R.PAIR_FNS
# kernel_cases' table plus a second nullable DOUBLE column e
SCHEMA = kc.SCHEMA + [("e", T.DOUBLE, True)]
COL = {name: i for i, (name, _, _) in enumerate(SCHEMA)}
TYPE = {name: t for name, t, _ in SCHEMA}
NULLABLE = {name: n for name, _, n in SCHEMA}
STORE_SCHEMA = [(t, n) for _, t, n in SCHEMA]


def cov_plan(keys, pairs=(("d", "e"),), filter_lit=False):
    """keys ++ [COUNT(*), SUM(x0), STDDEV(x0)] ++ [COVAR_POP, COVAR_SAMP, CORR] per (x, y) of `pairs` (x0: the first pair's x);
    non-DOUBLE inputs are cast as Spark casts them; filter `i IS NULL OR i > lit` when asked"""
    b = PlanBuilder()
    names = ["i"] + list(keys) + [n for p in pairs for n in p]
    e = {}
    for name in names:
        if name not in e:
            e[name] = b.col(TYPE[name], COL[name], NULLABLE[name])
    dbl = {name: e[name].cast(T.DOUBLE) for name in e}
    if filter_lit:
        b.filter(e["i"].is_null() | (e["i"] > b.lit(T.INT)))
    if keys:
        b.group_by(*[e[k] for k in keys])
    b.count().sum(dbl[pairs[0][0]]).stddev(dbl[pairs[0][0]])
    for x, y in pairs:
        b.covar_pop(dbl[x], dbl[y]).covar_samp(dbl[x], dbl[y]).corr(dbl[x], dbl[y])
    return b.build()


def profile_values(profile, g, rng):
    """(x, y) per row of group g"""
    n = len(g)
    z1, z2 = rng.standard_normal(n), rng.standard_normal(n)
    if profile == "big_mean_09":
        return 1e9 + z1, 1e9 + 0.9 * z1 + math.sqrt(0.19) * z2
    if profile == "big_mean_0":
        return 1e9 + z1, 1e9 + z2
    if profile == "big_mean_neg1":   # 2e9 - x is exact in x's binade: CORR is exactly -1
        x = 1e9 + z1
        return x, 2e9 - x
    if profile == "tiny":
        return 1e-6 * z1, 1e-6 * (0.9 * z1 + math.sqrt(0.19) * z2)
    sx, sy = 10.0 ** ((g % 7) - 2), 10.0 ** ((g % 5) - 3)   # groups of very different magnitudes in one table
    return 10.0 ** ((g % 5) * 2) + sx * z1, -(10.0 ** (g % 4)) + sy * (0.5 * z1 + z2)


def numeric_batch(n, kind, seed, groups, profile, batch_id=0, group_base=0, distinct_groups=False):
    """kernel_cases.make_batch with columns d, e holding the profile's x, y; e gets NULL runs of its own"""
    _, raw = kc.make_batch(n, kind, seed, groups, batch_id=batch_id, group_base=group_base, distinct_groups=distinct_groups)
    assert not raw.deltas and not len(raw.deletes)
    rng = np.random.default_rng(seed + 7)
    gid = np.array([int(k[1:]) if k[:1] == b"g" else int(k[3:]) for k in raw.values["k"]])
    raw.values["d"], raw.values["e"] = profile_values(profile, gid, rng)
    en = np.zeros(n, dtype=bool)
    if "d" in raw.nulls and raw.nulls["d"].any():   # the kinds with NULLs: runs of NULL y where x is set, and the reverse
        r = np.arange(n)
        en = ((r // 37) % 11 == 3) | (rng.random(n) < 0.05)
    raw.nulls["e"] = en
    batch = build_batch(n, SCHEMA, raw.values, raw.nulls, batch_id=batch_id, bucket_id=batch_id % 4, encoders=kc.ENCODERS[kind])
    batch.stats = None
    return batch, raw


def expected(keys, pairs, raws, lit=None):
    """{key tuple: {column: [values of the live rows that pass the filter, None for NULL]}}"""
    names = sorted({n for p in pairs for n in p})
    groups = {}
    for raw in raws:
        live = raw.live()
        cols = {name: raw.effective(name) for name in set(names) | {"i"} | set(keys)}
        for r in range(raw.n):
            if not live[r]:
                continue
            if lit is not None and not (cols["i"][1][r] or cols["i"][0][r] > lit):
                continue
            key = tuple(None if cols[k][1][r] else cols[k][0][r] for k in keys)
            g = groups.setdefault(key, {n: [] for n in names})
            for n in names:
                g[n].append(None if cols[n][1][r] else float(cols[n][0][r]))
    return groups


def exact_table(want, pairs):
    """{key: [(exact results, sqrt(varX varY)) per pair]} of expected()'s groups"""
    return {k: [R.exact_all(list(zip(g[x], g[y]))) for x, y in pairs] for k, g in want.items()}


def check(plan, keys, pairs, raws, raw_partials, lit=None, what="", want=None, exact=None):
    """final rows of the device's partial rows against exact arithmetic and against Spark's row-order update (`want` and
    `exact`: expected() and exact_table() of these batches, when already at hand)"""
    want = want if want is not None else expected(keys, pairs, raws, lit)
    exact = exact if exact is not None else exact_table(want, pairs)
    got = plan.final_merge(raw_partials)
    nk = len(keys)
    assert sorted(repr(tuple(r[:nk])) for r in got) == sorted(repr(k) for k in want), what
    worst = {fn: 0.0 for fn in FNS}
    for row in got:
        g = want[tuple(row[:nk])]
        xs0 = g[pairs[0][0]]
        assert row[nk] == len(xs0), what
        nn = [x for x in xs0 if x is not None]
        if row[nk + 1] is None or not all(math.isfinite(x) for x in nn):
            assert (row[nk + 1] is None) == (not nn), (what, row[:nk], row[nk + 1])
        else:
            assert abs(row[nk + 1] - math.fsum(nn)) <= 1e-12 * math.fsum(abs(x) for x in nn), (what, "sum", row[nk + 1])
        sd = MR.exact(AggFn.STDDEV_SAMP, xs0)
        assert MR.close(AggFn.STDDEV_SAMP, row[nk + 2], sd), (what, row[:nk], "stddev", row[nk + 2], sd)
        for p, (xn, yn) in enumerate(pairs):
            rows = list(zip(g[xn], g[yn]))
            exs, scale = exact[tuple(row[:nk])][p]
            for j, fn in enumerate(FNS):
                v = row[nk + 3 + 3 * p + j]
                ex = exs[fn]
                assert R.close(fn, v, ex, scale), (what, row[:nk], (xn, yn), fn, v, ex, scale)
                if ex is not None and not math.isnan(ex):
                    worst[fn] = max(worst[fn], abs(v - ex) / (1.0 if fn == AggFn.CORR else (scale or 1.0)))
                    sp = R.evaluate(fn, R.update(rows, fn == AggFn.CORR))   # Spark's row-order update, to its own rounding
                    assert (math.isnan(sp) and math.isnan(v)) or abs(sp - v) <= 1e-4 * max(scale if fn != AggFn.CORR else 1.0, abs(sp)), \
                        (what, fn, v, sp)
    print(what, len(got), "groups; worst error (covar: over sqrt(varX varY), corr: absolute)", worst)
    return want


def run(plan, batches, lits=(), store=None):
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
PROFILES = ["big_mean_09", "big_mean_0", "big_mean_neg1", "tiny", "mixed"]


@pytest.mark.parametrize("profile", PROFILES)
@pytest.mark.parametrize("accumulator", list(PLACEMENTS))
def test_placements_against_exact_arithmetic(gpu_api, monkeypatch, accumulator, profile):
    monkeypatch.setenv("SD_TUNE_CHUNK_ROWS", "2048")
    keys, groups = PLACEMENTS[accumulator]
    cases = [numeric_batch(n, kind, seed=500 + 10 * i + j, groups=groups, profile=profile, batch_id=2 * i + j)
             for i, n in enumerate((2049, 3 * 2048 + 77, 30000)) for j, kind in enumerate(("all_fast", "fast_nulls"))]
    batches, raws = [c[0] for c in cases], [c[1] for c in cases]
    pairs = (("d", "e"),)
    desc = cov_plan(keys, pairs, filter_lit=True)
    plan = capi.Plan(gpu_api, desc)
    st = capi.Store(gpu_api, STORE_SCHEMA)
    try:
        for b in batches:
            st.put(b)
        for lit in (-900, 200):   # one cached plan, new literals
            want = expected(keys, pairs, raws, lit)
            exact = exact_table(want, pairs)
            for where, store in (("submit", None), ("store", st)):
                raw = run(plan, batches, [lit], store)
                log = plan.launch_log()
                assert log and all(r["accumulator"] == accumulator for r in log), log
                check(plan, keys, pairs, raws, raw, lit, f"{accumulator}/{profile}/{where}/{lit}", want, exact)
        if profile.startswith("big_mean"):   # float64 raw sums of the same data miss the bar: the bar has teeth
            big = [list(zip(g["d"], g["e"])) for g in want.values() if len(R.counted(list(zip(g["d"], g["e"])))) > 100]
            assert any(not R.close(AggFn.COVAR_SAMP, R.naive(AggFn.COVAR_SAMP, r), R.exact(AggFn.COVAR_SAMP, r), R.exact_scale(r))
                       for r in big)
    finally:
        st.close()
        plan.close()


@pytest.mark.parametrize("kind", ["fast_overlay", "rle", "fast_nulls"])
def test_deltas_deletes_nulls_nan_and_infinity(gpu_api, monkeypatch, kind):
    """kernel_cases batches: update deltas and delete masks (overlay and per-row paths) in both inputs, NULL runs in either,
    and groups holding NaN / +-Inf (their results are NaN).  x = d, y = CAST(i AS DOUBLE); a second pair (CAST(f AS DOUBLE), d)."""
    monkeypatch.setenv("SD_TUNE_CHUNK_ROWS", "2048")
    cases = [kc.make_batch(n, kind, seed=60 + i, groups=9, batch_id=i) for i, n in enumerate(kc.BOUNDARY_SIZES)]
    batches = [c[0] for c in cases]
    pairs = (("d", "i"), ("f", "d"))
    for keys in ([], ["k"], ["h"]):
        desc = cov_plan(keys, pairs)
        plan = capi.Plan(gpu_api, desc)
        try:
            raw = run(plan, batches)
            want = check(plan, keys, pairs, [c[1] for c in cases], raw, None, f"{kind}/{keys}")
            if keys == ["k"]:
                assert any(any(x is not None and math.isnan(x) for x in g["d"]) for g in want.values())
        finally:
            plan.close()


def growth_batches():
    spec = [(100000, dict(groups=2)), (100000, dict(groups=100)), (100000, dict(groups=3000)),   # > 1 MB each: one launch each
            (75000, dict(groups=1, group_base=3000, distinct_groups=True))]
    return [numeric_batch(n, "fast_nulls", seed=877 + i, batch_id=i, profile="mixed", **kw) for i, (n, kw) in enumerate(spec)]


def test_placement_changes_hash_switch_and_grow(gpu_api, monkeypatch):
    """One execution of four launches: private -> shared-atomic -> global-atomic (the dense table re-indexed with its Kx / Ky
    words), then the switch to the hash table replays the earlier launches and the hash table grows and replays all four."""
    monkeypatch.setenv("SD_TUNE_FLUSH_MB", "1")
    cases = growth_batches()
    pairs = (("d", "e"),)
    desc = cov_plan(["k"], pairs)
    plan = capi.Plan(gpu_api, desc)
    try:
        raw = run(plan, [c[0] for c in cases[:3]])
        assert [r["accumulator"] for r in plan.launch_log()] == ["private", "shared_atomic", "global_atomic"]
        check(plan, ["k"], pairs, [c[1] for c in cases[:3]], raw, None, "growth dense")
        raw = run(plan, [c[0] for c in cases])
        seq = [(r["accumulator"], r["replay"]) for r in plan.launch_log()]
        assert seq[:3] == [("private", None), ("shared_atomic", None), ("global_atomic", None)], seq
        assert seq[3:7] == [("hash", "hash_switch")] * 3 + [("hash", None)], seq
        assert seq[7:] and all(s == ("hash", "hash_grow") for s in seq[7:]), seq
        check(plan, ["k"], pairs, [c[1] for c in cases], raw, None, "growth hash")
    finally:
        plan.close()


def test_no_rows_and_dense_partials_refused(gpu_api):
    desc = cov_plan([], filter_lit=True)
    plan = capi.Plan(gpu_api, desc)
    try:
        b, _ = numeric_batch(5000, "all_fast", seed=3, groups=4, profile="tiny")
        raw = run(plan, [b], [10 ** 6])                      # every row filtered out
        assert capi.parse_row_stream(raw, desc.partial_schema()) == [[0, None, 0.0, 0.0, 0.0] + [0.0] * 14]
        assert plan.final_merge(raw) == [[0, None, None, None, None, None]]
        import ctypes as C
        import torch
        lib, buf = gpu_api.lib, torch.zeros(4096, dtype=torch.float64, device="cuda")
        assert lib.sd_plan_partials_layout(plan.h, None, None, None) == capi.SD_ERR_UNSUPPORTED
        assert lib.sd_plan_export_partials(plan.h, C.c_void_p(buf.data_ptr()), C.c_int64(buf.numel() * 8)) == capi.SD_ERR_UNSUPPORTED
        assert lib.sd_plan_import_partials(plan.h, C.c_void_p(buf.data_ptr()), C.c_int64(22 * 8)) == capi.SD_ERR_UNSUPPORTED
        assert plan.final_merge(plan.finish_raw()) == [[0, None, None, None, None, None]]   # the refusals changed nothing
    finally:
        plan.close()


def test_exchange_on_two_gpus_equals_one_gpu():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29543", os.path.join(HERE, "covariance_multirank_worker.py")], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "COVARIANCE MULTIRANK OK" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])
