"""Spark 2.1.1 CentralMomentAgg restated in Python, for the moment-aggregate tests: Welford's update in row order, Chan's merge
and the evaluation of STDDEV_POP / STDDEV_SAMP / VAR_POP / VAR_SAMP / SKEWNESS / KURTOSIS; plus exact evaluation over
fractions.Fraction, the bar the device results are held to."""
import math
from fractions import Fraction
from typing import List, Optional, Sequence

from snappydata_b200.capi import AggFn

ORDER = {AggFn.STDDEV_POP: 2, AggFn.STDDEV_SAMP: 2, AggFn.VAR_POP: 2, AggFn.VAR_SAMP: 2, AggFn.SKEWNESS: 3, AggFn.KURTOSIS: 4}
MOMENT_FNS = tuple(ORDER)


def welford(xs: Sequence[Optional[float]], order: int) -> List[float]:
    """updateExpressions over the rows in order: the buffers [n, avg, m2, (m3, (m4))]; NULL (None) leaves them unchanged."""
    n = avg = m2 = m3 = m4 = 0.0
    for x in xs:
        if x is None:
            continue
        n1 = n + 1.0
        delta = x - avg
        dn = delta / n1
        avg = avg + dn
        m2n = m2 + delta * (delta - dn)
        if order >= 3:
            dn2 = dn * dn
            m3n = m3 - 3.0 * dn * m2n + delta * (delta * delta - dn2)
            if order >= 4:
                m4 = m4 - 4.0 * dn * m3n - 6.0 * dn2 * m2n + delta * (delta * delta * delta - dn * dn2)
            m3 = m3n
        n, m2 = n1, m2n
    return [n, avg, m2, m3, m4][: order + 1]


def merge(a: Sequence[float], b: Sequence[float], order: int) -> List[float]:
    """mergeExpressions of two buffers."""
    n1, n2 = a[0], b[0]
    n = n1 + n2
    delta = b[1] - a[1]
    dn = 0.0 if n == 0 else delta / n
    out = [n, a[1] + dn * n2, a[2] + b[2] + delta * dn * n1 * n2]
    if order >= 3:
        out.append(a[3] + b[3] + dn * dn * delta * n1 * n2 * (n1 - n2) + 3.0 * dn * (n1 * b[2] - n2 * a[2]))
    if order >= 4:
        out.append(a[4] + b[4] + dn * dn * dn * delta * n1 * n2 * (n1 * n1 - n1 * n2 + n2 * n2) +
                   6.0 * dn * dn * (n1 * n1 * b[2] + n2 * n2 * a[2]) + 4.0 * dn * (n1 * b[3] - n2 * a[3]))
    return out


def evaluate(fn: int, buf: Sequence[float]) -> Optional[float]:
    """evaluateExpression: NULL without input."""
    n, m2 = buf[0], buf[2]
    if n == 0:
        return None
    if fn == AggFn.VAR_POP:
        return m2 / n
    if fn == AggFn.STDDEV_POP:
        return math.sqrt(m2 / n)
    if fn in (AggFn.VAR_SAMP, AggFn.STDDEV_SAMP):
        if n == 1:
            return math.nan
        v = m2 / (n - 1.0)
        return v if fn == AggFn.VAR_SAMP else math.sqrt(v)
    if m2 == 0:
        return math.nan
    if fn == AggFn.SKEWNESS:
        return math.sqrt(n) * buf[3] / math.sqrt(m2 * m2 * m2)
    return n * buf[4] / (m2 * m2) - 3.0


def exact_moments(xs: Sequence[Optional[float]]):
    """(n, mean, m2, m3, m4) over the non-null values, exactly."""
    vals = [Fraction(x) for x in xs if x is not None]
    n = len(vals)
    if n == 0:
        return 0, Fraction(0), Fraction(0), Fraction(0), Fraction(0)
    mean = sum(vals, Fraction(0)) / n
    d = [v - mean for v in vals]
    return n, mean, sum((x * x for x in d), Fraction(0)), sum((x ** 3 for x in d), Fraction(0)), sum((x ** 4 for x in d), Fraction(0))


def exact(fn: int, xs: Sequence[Optional[float]]) -> Optional[float]:
    """The result of fn over the values as exact arithmetic gives it, rounded once to a double at the end."""
    vals = [x for x in xs if x is not None]
    if not vals:
        return None
    if any(math.isnan(x) or math.isinf(x) for x in vals):
        return math.nan
    n, _, m2, m3, m4 = exact_moments(vals)
    if fn == AggFn.VAR_POP:
        return float(m2 / n)
    if fn == AggFn.STDDEV_POP:
        return math.sqrt(float(m2 / n))
    if fn in (AggFn.VAR_SAMP, AggFn.STDDEV_SAMP):
        if n == 1:
            return math.nan
        v = m2 / (n - 1)
        return float(v) if fn == AggFn.VAR_SAMP else math.sqrt(float(v))
    if m2 == 0:
        return math.nan
    if fn == AggFn.SKEWNESS:
        return math.sqrt(n) * float(m3) / math.sqrt(float(m2)) ** 3
    return float(n * m4 / (m2 * m2)) - 3.0


def close(fn: int, got: Optional[float], want: Optional[float]) -> bool:
    """The bars: VAR / STDDEV within 1e-8 relative; SKEWNESS / KURTOSIS within 1e-6 relative, or 1e-9 absolute near 0."""
    if want is None or got is None:
        return got is None and want is None
    if math.isnan(want) or math.isnan(got):
        return math.isnan(want) and math.isnan(got)
    if fn in (AggFn.SKEWNESS, AggFn.KURTOSIS):
        return abs(got - want) <= max(1e-6 * abs(want), 1e-9)
    return abs(got - want) <= 1e-8 * abs(want) or got == want


def naive(fn: int, xs: Sequence[Optional[float]]) -> Optional[float]:
    """The same functions from float64 power sums sum x^j: what the shifted sums replace (it loses every digit when
    the mean is large against the spread)."""
    vals = [x for x in xs if x is not None]
    n = float(len(vals))
    if not vals:
        return None
    s1, s2, s3, s4 = sum(vals), sum(x * x for x in vals), sum(x ** 3 for x in vals), sum(x ** 4 for x in vals)
    mean = s1 / n
    m2 = s2 - n * mean * mean
    m3 = s3 - 3 * mean * s2 + 2 * n * mean ** 3
    m4 = s4 - 4 * mean * s3 + 6 * mean * mean * s2 - 3 * n * mean ** 4
    return evaluate(fn, [n, mean, m2, m3, m4])
