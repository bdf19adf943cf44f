"""The exact evaluator of tests/kernel_cases.py against the CPU oracle, before it is used to judge the kernel: on every
scenario the partial rows must be equal field for field (doubles bit for bit), and the final DECIMAL averages must be
the oracle's HALF_UP quotients."""
import math

import pytest

from oracle import oracle
from snappydata_b200.capi import AggFn

import kernel_cases as kc


def run_oracle(query, batches):
    pl = oracle.plan(query.desc()).set_literals(query.literals())
    for b in batches:
        pl.submit(b)
    raw = pl.finish_raw()
    rows = pl.finish()
    pl.close()
    return rows, raw


QUERIES = {
    "string_key": kc.Query(["k"], kc.EVERY_AGG, filter_lit=-900),
    "no_key": kc.Query([], kc.EVERY_AGG, filter_lit=-900),
    "int_key": kc.Query(["h"], [(AggFn.COUNT_STAR, None), (AggFn.SUM, "d"), (AggFn.AVG, "m"), (AggFn.MIN, "s"),
                                (AggFn.MAX, "d"), (AggFn.SUM, "l")]),
}


@pytest.mark.parametrize("kind", kc.KINDS)
def test_evaluator_equals_oracle_on_every_batch_kind(oracle_api, kind):
    cases = [kc.make_batch(n, kind, seed=1000 + i, groups=9, batch_id=i) for i, n in enumerate(kc.BOUNDARY_SIZES)]
    batches, raws = [c[0] for c in cases], [c[1] for c in cases]
    for name, q in QUERIES.items():
        got, _ = run_oracle(q, batches)
        want = kc.evaluate(q, raws)
        kc.assert_rows_exact(got, want, q, f"{kind}/{name}")


def test_special_value_groups_follow_their_rule(oracle_api):
    """NaN wins MAX and poisons SUM, +inf with -inf sums to NaN, +-0.0 only sums to +0.0, all-NULL gives NULL."""
    cases = [kc.make_batch(4000, "fast_nulls", seed=7, groups=8)]
    q = kc.Query(["k"], [(AggFn.SUM, "d"), (AggFn.MIN, "d"), (AggFn.MAX, "d"), (AggFn.COUNT, "d")])
    rows = {r[0]: r[1:] for r in kc.evaluate(q, [cases[0][1]])}
    got, _ = run_oracle(q, [cases[0][0]])
    kc.assert_rows_exact(got, list([k] + v for k, v in rows.items()), q)
    s, mn, mx, cnt = rows[kc.key_of(1)]
    assert math.isnan(s) and math.isnan(mx) and not math.isnan(mn)
    assert rows[kc.key_of(2)][0] == math.inf and rows[kc.key_of(6)][0] == -math.inf
    assert math.isnan(rows[kc.key_of(3)][0])
    s, mn, mx, cnt = rows[kc.key_of(4)]
    assert s == 0.0 and str(s) == "0.0" and mn == 0.0 and mx == 0.0 and cnt > 0
    assert rows[kc.key_of(5)] == [None, None, None, 0]


def test_long_sum_wraps_and_decimal_halves_carry(oracle_api):
    cases = [kc.make_batch(20000, "all_fast", seed=11, groups=3)]
    q = kc.Query([], [(AggFn.SUM, "l"), (AggFn.SUM, "m"), (AggFn.AVG, "m")])
    (want,) = kc.evaluate(q, [cases[0][1]])
    exact_l = sum(int(x) for x in cases[0][1].values["l"].tolist())
    assert exact_l > (1 << 63) and want[0] == kc._wrap64(exact_l)     # the LONG sum wrapped
    lo = sum(int(x) & 0xFFFFFFFF for x in cases[0][1].values["m"].tolist())
    assert lo >= (1 << 40)                                              # low halves carry far past 2^32
    got, raw = run_oracle(q, [cases[0][0]])
    kc.assert_rows_exact(got, [want], q)
    final = oracle.final_merge(q.desc(), raw)
    assert final[0][2] == kc.decimal_avg_half_up(want[2], want[3]) == kc.final_rows(q, [want])[0][2]


def test_decimal_average_rounds_half_up_away_from_zero():
    assert kc.decimal_avg_half_up(5, 20000) == 3            # 2.5 -> 3
    assert kc.decimal_avg_half_up(-5, 20000) == -3          # -2.5 -> -3
    assert kc.decimal_avg_half_up(1, 30000) == 0            # 0.333.. -> 0
    assert kc.decimal_avg_half_up(7, 0) is None
