"""Spark 2.1.1 Covariance / Corr restated in Python, for the two-input aggregate tests: the row-order update, the merge and the
evaluation of COVAR_POP / COVAR_SAMP / CORR; plus exact evaluation over fractions.Fraction, the bar the device results are held
to.  Restated from upstream Spark 2.1.1 (catalyst/expressions/aggregate/Covariance.scala, Corr.scala)."""
import math
from fractions import Fraction
from typing import List, Optional, Sequence, Tuple

from snappydata_b200.capi import AggFn

FIELDS = {AggFn.COVAR_POP: 4, AggFn.COVAR_SAMP: 4, AggFn.CORR: 6}
PAIR_FNS = tuple(FIELDS)
Pair = Tuple[Optional[float], Optional[float]]


def update(rows: Sequence[Pair], corr: bool = True) -> List[float]:
    """updateExpressions over the rows in order: the buffers [n, xAvg, yAvg, ck, (xMk, yMk)]; a row with a NULL (None) in x or
    y leaves them unchanged."""
    n = x_avg = y_avg = ck = x_mk = y_mk = 0.0
    for x, y in rows:
        if x is None or y is None:
            continue
        new_n = n + 1.0
        dx = x - x_avg
        dy = y - y_avg
        x_avg = x_avg + dx / new_n
        y_avg = y_avg + dy / new_n
        ck = ck + dx * (y - y_avg)
        if corr:
            x_mk = x_mk + dx * (x - x_avg)
            y_mk = y_mk + dy * (y - y_avg)
        n = new_n
    out = [n, x_avg, y_avg, ck, x_mk, y_mk]
    return out if corr else out[:4]


def merge(a: Sequence[float], b: Sequence[float]) -> List[float]:
    """mergeExpressions of two buffers (four or six fields)."""
    n1, n2 = a[0], b[0]
    n = n1 + n2
    dx, dy = b[1] - a[1], b[2] - a[2]
    dxn = 0.0 if n == 0 else dx / n
    dyn = 0.0 if n == 0 else dy / n
    out = [n, a[1] + dxn * n2, a[2] + dyn * n2, a[3] + b[3] + dx * dyn * n1 * n2]
    if len(a) == 6:
        out += [a[4] + b[4] + dx * dxn * n1 * n2, a[5] + b[5] + dy * dyn * n1 * n2]
    return out


def jdiv(a: float, b: float) -> float:
    """a / b as Java doubles divide: x / 0 is +-Inf, 0 / 0 and NaN / 0 are NaN."""
    if b != 0 or math.isnan(b):
        return a / b
    if a == 0 or math.isnan(a):
        return math.nan
    return math.copysign(math.inf, a) * math.copysign(1.0, b)


def jsqrt(v: float) -> float:
    """java.lang.Math.sqrt: NaN below 0."""
    return math.nan if v < 0 or math.isnan(v) else math.sqrt(v)


def evaluate(fn: int, buf: Sequence[float]) -> Optional[float]:
    """evaluateExpression: NULL without input."""
    n, ck = buf[0], buf[3]
    if n == 0:
        return None
    if fn == AggFn.COVAR_POP:
        return ck / n
    if n == 1:
        return math.nan
    if fn == AggFn.COVAR_SAMP:
        return ck / (n - 1.0)
    return jdiv(ck, jsqrt(buf[4] * buf[5]))


def counted(rows: Sequence[Pair]) -> List[Tuple[float, float]]:
    return [(x, y) for x, y in rows if x is not None and y is not None]


def exact_buffers(rows: Sequence[Pair]):
    """(n, xMean, yMean, ck, xMk, yMk) over the counted rows, exactly (finite values only)."""
    vals = [(Fraction(x), Fraction(y)) for x, y in counted(rows)]
    n = len(vals)
    if n == 0:
        return 0, Fraction(0), Fraction(0), Fraction(0), Fraction(0), Fraction(0)
    mx = sum((x for x, _ in vals), Fraction(0)) / n
    my = sum((y for _, y in vals), Fraction(0)) / n
    ck = sum(((x - mx) * (y - my) for x, y in vals), Fraction(0))
    return n, mx, my, ck, sum(((x - mx) ** 2 for x, _ in vals), Fraction(0)), sum(((y - my) ** 2 for _, y in vals), Fraction(0))


def exact(fn: int, rows: Sequence[Pair]) -> Optional[float]:
    """The result of fn over the rows as exact arithmetic gives it, rounded once to a double at the end (square root of the
    rounded quotient for CORR)."""
    vals = counted(rows)
    if not vals:
        return None
    if any(not math.isfinite(v) for r in vals for v in r):
        return math.nan
    n, _, _, ck, xmk, ymk = exact_buffers(vals)
    if fn == AggFn.COVAR_POP:
        return float(ck / n)
    if n == 1:
        return math.nan
    if fn == AggFn.COVAR_SAMP:
        return float(ck / (n - 1))
    if xmk == 0 or ymk == 0:
        return math.nan
    s = 1.0 if ck >= 0 else -1.0
    return s * math.sqrt(float(ck * ck / (xmk * ymk)))


def exact_all(rows: Sequence[Pair]):
    """({fn: exact(fn, rows)}, exact_scale(rows)) from one exact pass over the rows."""
    vals = counted(rows)
    if not vals:
        return {fn: None for fn in PAIR_FNS}, 0.0
    if any(not math.isfinite(v) for r in vals for v in r):
        return {fn: math.nan for fn in PAIR_FNS}, 0.0
    n, _, _, ck, xmk, ymk = exact_buffers(vals)
    out = {AggFn.COVAR_POP: float(ck / n)}
    if n == 1:
        out[AggFn.COVAR_SAMP] = out[AggFn.CORR] = math.nan
    else:
        out[AggFn.COVAR_SAMP] = float(ck / (n - 1))
        out[AggFn.CORR] = math.nan if xmk == 0 or ymk == 0 else (1.0 if ck >= 0 else -1.0) * math.sqrt(float(ck * ck / (xmk * ymk)))
    return out, math.sqrt(float(xmk / n) * float(ymk / n))


def exact_scale(rows: Sequence[Pair]) -> float:
    """sqrt(varX * varY) (population variances) of the counted rows: the covariance bar's unit."""
    vals = counted(rows)
    if not vals or any(not math.isfinite(v) for r in vals for v in r):
        return 0.0
    n, _, _, _, xmk, ymk = exact_buffers(vals)
    return math.sqrt(float(xmk / n) * float(ymk / n))


def close(fn: int, got: Optional[float], want: Optional[float], scale: float) -> bool:
    """The bars: |covar - exact| <= 1e-8 * sqrt(varX * varY); |corr - exact| <= 1e-8."""
    if want is None or got is None:
        return got is None and want is None
    if math.isnan(want) or math.isnan(got):
        return math.isnan(want) and math.isnan(got)
    if fn == AggFn.CORR:
        return abs(got - want) <= 1e-8
    return abs(got - want) <= 1e-8 * scale or got == want


def naive(fn: int, rows: Sequence[Pair]) -> Optional[float]:
    """The same functions from float64 raw sums sum x, sum y, sum xy (sum x^2, sum y^2): what the shifted sums replace (it loses
    every digit when the means are large against the spreads)."""
    vals = counted(rows)
    if not vals:
        return None
    n = float(len(vals))
    sx, sy = sum(x for x, _ in vals), sum(y for _, y in vals)
    sxy, sxx, syy = sum(x * y for x, y in vals), sum(x * x for x, _ in vals), sum(y * y for _, y in vals)
    mx, my = sx / n, sy / n
    return evaluate(fn, [n, mx, my, sxy - n * mx * my, sxx - n * mx * mx, syy - n * my * my])
