"""GROUP BY ... WITH ROLLUP / WITH CUBE / GROUPING SETS through CUDA: the scan runs the plain GROUP BY's kernel once and the
roll-up kernel (sd_rollup.cu) combines its groups into every set.  Checked against the reference's closed forms, against Expand
restated per set on the CPU oracle and on the existing engine (one plain GROUP BY per set), per placement of the scan's group
table, for moment and covariance aggregates on data whose mean dwarfs its spread, and through the roll-up table's growth."""
import math

import numpy as np
import pytest

import grouping_sets_cases as G
import kernel_cases as kc
import known_answer_cases as K
import covariance_reference as CR
import moments_reference as R
import test_gpu_covariance as CV
from snappydata_b200 import capi
from snappydata_b200.capi import AggFn
from snappydata_b200.column_format import (ColumnBatch, SqlType as T, build_batch, encode_column, encode_uncompressed,
                                           encode_wide_decimal)
from snappydata_b200.plan import PlanBuilder, q1_plan, Q1_LITERALS

pytestmark = pytest.mark.gpu

AGGS = [(AggFn.COUNT_STAR, None), (AggFn.SUM, "i"), (AggFn.SUM, "d"), (AggFn.AVG, "m"), (AggFn.MIN, "s"), (AggFn.MAX, "s"),
        (AggFn.MIN, "d"), (AggFn.MAX, "l"), (AggFn.SUM, "m")]


def _desc(keys, shape, aggs=AGGS, sets=None):
    b = PlanBuilder()
    used = set(keys) | {c for _, c in aggs if c}
    e = {n: b.col(kc.TYPE[n], kc.COL[n], kc.NULLABLE[n], scale=kc.DEC_SCALE if kc.TYPE[n] == T.DECIMAL else 0)
         for n, _, _ in kc.SCHEMA if n in used}
    ks = [e[k] for k in keys]
    if shape == "rollup":
        b.rollup(*ks)
    elif shape == "cube":
        b.cube(*ks)
    else:
        b.grouping_sets(ks, [[e[k] for k in st] for st in sets])
    for fn, c in aggs:
        b.agg(fn, e[c] if c else None)
    return b.build()


def _close_rows(got, want, nkeys, what=""):
    key = lambda r: repr(r[:nkeys])
    got, want = sorted(got, key=key), sorted(want, key=key)
    assert [key(r) for r in got] == [key(r) for r in want], what
    for g, w in zip(got, want):
        for a, b in zip(g[nkeys:], w[nkeys:]):
            if isinstance(a, float) or isinstance(b, float):
                assert (math.isnan(a) and math.isnan(b)) or abs(a - b) <= 1e-6 * max(abs(a), abs(b)) or a == b, (what, g, w)
            else:
                assert a == b, (what, g, w)


def _gpu_rows(api, desc, batches, lits=()):
    pl = capi.Plan(api, desc).set_literals(list(lits))
    for b in batches:
        pl.submit(b)
    raw = pl.finish_raw()
    return capi.final_merge(api, desc, raw), pl


# ---- closed forms ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", G.CLOSED_FORMS, ids=lambda c: c.__name__)
def test_closed_form_on_gpu(case, gpu_api):
    case(K.GpuEngine(gpu_api))


# ---- every placement of the scan's table, against Expand on the oracle and on the existing engine ---------------------------
# placement -> (keys, groups drawn, accumulator of the scan)
# (each dense placement and both replays are pinned one by one in test_every_placement_and_replay_pinned)
DENSE = {"private", "shared_atomic", "global_atomic"}
PLACEMENTS = {"dense": (["k", "s"], 300, DENSE), "hash": (["h", "i", "m"], 300, {"hash"})}
SHAPES = {"rollup": None, "cube": None, "sets": "explicit"}


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("placement", list(PLACEMENTS))
def test_placements_against_expand(gpu_api, oracle_api, monkeypatch, placement, shape):
    monkeypatch.setenv("SD_TUNE_CHUNK_ROWS", "2048")
    keys, groups, acc = PLACEMENTS[placement]
    # batches with different dictionaries (group_base shifts the key values each batch draws)
    batches = [kc.make_batch(5000 + 777 * j, kind, 40 + j, groups, batch_id=j, group_base=j)[0]
               for j, kind in enumerate(["fast_nulls", "dictionary", "all_fast"])]
    sets = [[keys[0]], [], keys[1:]] if shape == "sets" else None   # includes (), omits the finest set
    desc = _desc(keys, shape, sets=sets)
    got, pl = _gpu_rows(gpu_api, desc, batches)
    log = pl.launch_log()
    assert len({l["accumulator"] for l in log}) == 1 and {l["accumulator"] for l in log} <= acc, log
    n = len(keys) + 1
    want_gpu = G.expand_reference(K.GpuEngine(gpu_api), desc, [], batches)
    _close_rows(got, want_gpu, n, "vs plain GROUP BY per set on the GPU")
    want_oracle = G.expand_reference(K.OracleEngine(oracle_api), desc, [], batches)
    _close_rows(got, want_oracle, n, "vs Expand on the oracle")
    assert {r[len(keys)] for r in got} == set(G.split(desc)[1])
    # the scan is the plain GROUP BY's: same kernel, same launches
    plain = G.set_plan(desc, 0)
    _, pp = _gpu_rows(gpu_api, plain, batches)
    assert pp.kernel_name() == pl.kernel_name()
    assert pp.launch_log() == log
    pl.close(); pp.close()


# ---- the ahead-of-time Q1 kernel -----------------------------------------------------------------------------------------
def test_rollup_q1_runs_the_aot_kernel(gpu_api):
    from snappydata_b200 import lineitem
    from snappydata_b200.capi import Op, PlanDesc
    d = q1_plan()
    first = len(d.exprs_py)
    nodes = [(Op.GROUPING_SET, int(T.INT), m, 0, 0) for m in (0, 1, 3)] + [(Op.GROUPING_ID, int(T.INT), first, 3, 0)]
    desc = PlanDesc(d.cols_py, d.exprs_py + nodes, d.filter, d.keys_py + [first + 3], d.aggs_py, d.proj_py, d.literal_types_py)
    batches = lineitem.gen_table(total_rows=60_000, rows_per_batch=20_000, seed=3)
    got, pl = _gpu_rows(gpu_api, desc, batches, Q1_LITERALS)
    assert pl.kernel_name().startswith("aot:")
    want = G.expand_reference(K.GpuEngine(gpu_api), desc, Q1_LITERALS, batches)
    _close_rows(got, want, 3)
    info = pl.rollup_info()
    assert info["launches"] == 1 and info["coarse"] == len(got) and info["fine"] == len([r for r in got if r[2] == 0])


# ---- growth of the roll-up table --------------------------------------------------------------------------------------------
def test_rollup_table_grows_without_replaying_the_scan(gpu_api, monkeypatch):
    monkeypatch.setenv("SD_TUNE_ROLLUP_CAP", "16")
    batches = [kc.make_batch(20000, "all_fast", 90 + j, 20000, batch_id=j, distinct_groups=True, group_base=20000 * j)[0]
               for j in range(2)]
    desc = _desc(["h", "l"], "rollup", aggs=[(AggFn.COUNT_STAR, None), (AggFn.SUM, "d")])
    got, pl = _gpu_rows(gpu_api, desc, batches)
    info = pl.rollup_info()
    assert info["launches"] > 1 and info["coarse"] == len(got), info
    _, pp = _gpu_rows(gpu_api, G.set_plan(desc, 0), batches)
    assert pl.launch_log() == pp.launch_log()   # the roll-up re-ran alone: the scan's launches are the plain GROUP BY's
    monkeypatch.delenv("SD_TUNE_ROLLUP_CAP")
    want = G.expand_reference(K.GpuEngine(gpu_api), desc, [], batches)
    _close_rows(got, want, 3)


def test_no_rows_no_output(gpu_api):
    rows, _ = K.GpuEngine(gpu_api)(G.mytable_plan("cube"), [], [])
    assert rows == []


# ---- every placement and replay, pinned, with moments and covariance of two inputs and NaN rows -----------------------------
def _cov_batch(n, seed, batch_id, **kw):
    """test_gpu_covariance's table (d, e = x, y at mean 1e9, sigma 1, correlation 0.9) with NaN in d for every row of the
    groups g % 7 == 3"""
    _, raw = kc.make_batch(n, "fast_nulls", seed, batch_id=batch_id, **kw)
    rng = np.random.default_rng(seed + 7)
    g = np.array([int(k[1:]) if k[:1] == b"g" else int(k[3:]) for k in raw.values["k"]])
    raw.values["d"], raw.values["e"] = CV.profile_values("big_mean_09", g, rng)
    raw.values["d"] = np.where(g % 7 == 3, np.nan, raw.values["d"])
    raw.nulls["e"] = (np.arange(n) // 37) % 11 == 3
    batch = build_batch(n, CV.SCHEMA, raw.values, raw.nulls, batch_id=batch_id)
    batch.stats = None
    return batch, raw


def _pinned_plan():
    b = PlanBuilder()
    e = {n: b.col(CV.TYPE[n], CV.COL[n], CV.NULLABLE[n]) for n in ("k", "d", "e")}
    b.rollup(e["k"])
    b.count().var_samp(e["d"]).kurtosis(e["d"]).covar_pop(e["d"], e["e"]).corr(e["d"], e["e"])
    return b.build()


def _check_pinned(got, raws):
    want = {}
    for m, present in ((0, ["k"]), (1, [])):
        for key, g in CV.expected(present, (("d", "e"),), raws).items():
            want[(key[0] if key else None, m)] = g
    assert sorted(repr(tuple(r[:2])) for r in got) == sorted(repr(k) for k in want)
    nan_groups = 0
    for r in got:
        g = want[tuple(r[:2])]
        xs, pairs = g["d"], list(zip(g["d"], g["e"]))
        assert r[2] == len(xs)
        for fn, v in ((AggFn.VAR_SAMP, r[3]), (AggFn.KURTOSIS, r[4])):
            assert R.close(fn, v, R.exact(fn, xs)), (r[:2], fn, v)
        exact, scale = CR.exact_all(pairs)
        for fn, v in ((AggFn.COVAR_POP, r[5]), (AggFn.CORR, r[6])):
            assert CR.close(fn, v, exact[fn], scale), (r[:2], fn, v, exact[fn])
        nan_groups += r[3] is not None and math.isnan(r[3])
    assert nan_groups > 0   # groups with NaN rows (the () group among them) give NaN


def test_every_placement_and_replay_pinned(gpu_api, monkeypatch):
    """ROLLUP(k) over one execution of three launches, private -> shared-atomic -> global-atomic, then over one of four: the
    dense table switches to the hash table (the first three replayed) and the hash table grows (all four replayed).  The
    roll-up reads the dense table's K words in the first, the hash entries' in the second; the scan's launches are the plain
    GROUP BY's."""
    monkeypatch.setenv("SD_TUNE_FLUSH_MB", "1")
    spec = [(100000, dict(groups=2)), (100000, dict(groups=100)), (100000, dict(groups=3000)),
            (75000, dict(groups=1, group_base=3000, distinct_groups=True))]
    cases = [_cov_batch(n, 777 + i, i, **kw) for i, (n, kw) in enumerate(spec)]
    desc = _pinned_plan()
    got, pl = _gpu_rows(gpu_api, desc, [c[0] for c in cases[:3]])
    assert [r["accumulator"] for r in pl.launch_log()] == ["private", "shared_atomic", "global_atomic"]
    _check_pinned(got, [c[1] for c in cases[:3]])
    _, pp = _gpu_rows(gpu_api, G.set_plan(desc, 0), [c[0] for c in cases[:3]])
    assert pp.launch_log() == pl.launch_log()
    got, pl = _gpu_rows(gpu_api, desc, [c[0] for c in cases])
    seq = [(r["accumulator"], r["replay"]) for r in pl.launch_log()]
    assert seq[:3] == [("private", None), ("shared_atomic", None), ("global_atomic", None)], seq
    assert seq[3:7] == [("hash", "hash_switch")] * 3 + [("hash", None)], seq
    assert seq[7:] and all(x == ("hash", "hash_grow") for x in seq[7:]), seq
    _check_pinned(got, [c[1] for c in cases])


# ---- keys held by reference: raw STRING and DECIMAL(38, 2) ---------------------------------------------------------------------
WORDS = [b"", b"a", b"ab", b"abc", b"zeta", b"\xc3\xa9t\xc3\xa9", b"a" * 40]
WIDE = [0, 10 ** 30 + 7, -(10 ** 35), 123456789012345678901234567, -5]


def _ref_batch(n, seed, batch_id, raw_strings):
    """s STRING (a dictionary of its own order per batch, or raw [len][bytes] records), w DECIMAL(38, 2), v LONG, t STRING"""
    r = np.random.default_rng(seed)
    words = [WORDS[i] for i in r.permutation(len(WORDS))]   # dictionary order differs between batches
    s = [words[i] for i in r.integers(0, len(words), n)]
    t = [b"t%d" % i for i in r.integers(0, 5, n)]
    w = [WIDE[i] for i in r.integers(0, len(WIDE), n)]
    v = r.integers(-1000, 1000, n).astype(np.int64)
    sn, wn = r.random(n) < 0.1, r.random(n) < 0.1
    enc = (lambda vals, nulls: encode_uncompressed(np.array(vals, dtype=object), T.STRING, nulls)) if raw_strings else \
          (lambda vals, nulls: encode_column(np.array(vals, dtype=object), T.STRING, nulls))
    cols = [enc(s, sn), encode_wide_decimal(w, wn), encode_uncompressed(v, T.LONG),
            enc(t, None)]
    rows = [(None if sn[i] else s[i], None if wn[i] else w[i], int(v[i]), t[i]) for i in range(n)]
    return ColumnBatch(num_rows=n, columns=cols, stats=None, batch_id=batch_id), rows


def _ref_plan(keys, shape):
    b = PlanBuilder()
    s, w, v, t = (b.col(T.STRING, 0, True), b.col(T.DECIMAL, 1, True, scale=2, precision=38), b.col(T.LONG, 2, False),
                  b.col(T.STRING, 3, False))
    e = {"s": s, "w": w, "t": t}
    (b.rollup if shape == "rollup" else b.cube)(*[e[k] for k in keys])
    b.count().sum(v).sum(w).min(w).max(w).min(s).max(s)
    return b.build()


def _ref_expected(keys, masks, rows):
    """(keys, gid, COUNT(*), SUM(v), SUM(w), MIN(w), MAX(w), MIN(s), MAX(s)) per coarse group, exactly"""
    col = {"s": 0, "w": 1, "t": 3}
    n, out = len(keys), {}
    for m in masks:
        for r in rows:
            key = tuple(None if (m >> (n - 1 - i)) & 1 else r[col[k]] for i, k in enumerate(keys)) + (m,)
            g = out.setdefault(key, [0, 0, None, None, None, None, None])
            g[0] += 1
            g[1] += r[2]
            if r[1] is not None:
                g[2] = r[1] if g[2] is None else g[2] + r[1]
                g[3] = r[1] if g[3] is None else min(g[3], r[1])
                g[4] = r[1] if g[4] is None else max(g[4], r[1])
            if r[0] is not None:
                g[5] = r[0] if g[5] is None else min(g[5], r[0])
                g[6] = r[0] if g[6] is None else max(g[6], r[0])
    for v in out.values():   # SUM's buffer is DECIMAL(38, 2): a total of more than 38 digits is NULL
        if v[2] is not None and abs(v[2]) >= 10 ** 38:
            v[2] = None
    return sorted((list(k) + v for k, v in out.items()), key=lambda x: repr(x[:n + 1]))


@pytest.mark.parametrize("shape", ["rollup", "cube"])
def test_raw_string_and_wide_decimal_keys(gpu_api, shape):
    """CUBE / ROLLUP(s, w): STRING and DECIMAL(38, 2) keys held by record address, compared by their bytes -- equal values of
    different batches (dictionary and raw bodies) are different fine groups and meet in one coarse group; SUM / MIN / MAX of the
    wide DECIMAL, MIN / MAX of the STRING"""
    parts = [_ref_batch(4000, 10 + j, j, raw_strings=j % 2 == 1) for j in range(4)]
    desc = _ref_plan(["s", "w"], shape)
    got, pl = _gpu_rows(gpu_api, desc, [p[0] for p in parts])
    assert {l["accumulator"] for l in pl.launch_log()} == {"hash"}
    want = _ref_expected(["s", "w"], G.split(desc)[1], [r for p in parts for r in p[1]])
    assert sorted(got, key=lambda x: repr(x[:3])) == want
    info = pl.rollup_info()
    assert info["coarse"] == len(want) and info["fine"] == sum(1 for r in want if r[2] == 0)
    _close_rows(got, G.expand_reference(K.GpuEngine(gpu_api), desc, [], [p[0] for p in parts]), 3, "vs plain GROUP BY per set")


def test_dictionary_then_raw_string_keys_switch_and_replay(gpu_api, monkeypatch):
    """ROLLUP(s, t) over dictionary batches, then raw ones: the dense table gives way to the hash table (the earlier launches
    replayed) and the roll-up compares the keys by their bytes"""
    monkeypatch.setenv("SD_TUNE_FLUSH_MB", "1")
    parts = [_ref_batch(60000, 30 + j, j, raw_strings=j >= 2) for j in range(4)]
    desc = _ref_plan(["s", "t"], "rollup")
    got, pl = _gpu_rows(gpu_api, desc, [p[0] for p in parts])
    seq = [(r["accumulator"], r["replay"]) for r in pl.launch_log()]
    assert seq[0][0] in DENSE and ("hash", "hash_switch") in seq, seq
    want = _ref_expected(["s", "t"], G.split(desc)[1], [r for p in parts for r in p[1]])
    assert sorted(got, key=lambda x: repr(x[:3])) == want
