"""Spark 2.1.1 First / Last, restated from upstream Spark (the fork's sources are not in the reference checkout), twice:

  * `update_rows` walks the rows in scan order and applies the update rule of First.scala / Last.scala row by row:
      FIRST  value = valueSet ? value : x,  valueSet = true
      LAST   value = x,                     valueSet = true
    with ignoreNulls only the rows whose x is not NULL count;
  * `numpy_rows` finds the first / last qualifying position of every group with numpy, independently of that loop.

Both produce partial rows (keys ++ [value, valueSet] per aggregate, the buffers sd_plan_finish emits) over the batches of
tests/kernel_cases.py: effective value = depth-0 delta, else depth-1 delta, else base; deleted rows dropped; the filter
`i > lit` (when given) rejects rows.  `merge` is Spark's merge of two partial buffers.  None of this calls the product."""
import math
import struct
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

import kernel_cases as kc
from snappydata_b200.capi import AggFn
from snappydata_b200.column_format import SqlType as T
from snappydata_b200.plan import PlanBuilder

ORDER_FNS = (AggFn.FIRST, AggFn.LAST, AggFn.FIRST_IGNORE_NULLS, AggFn.LAST_IGNORE_NULLS)


def is_last(fn) -> bool:
    return fn in (AggFn.LAST, AggFn.LAST_IGNORE_NULLS)


def ignores_nulls(fn) -> bool:
    return fn in (AggFn.FIRST_IGNORE_NULLS, AggFn.LAST_IGNORE_NULLS)


def desc(keys: Sequence[str], aggs: Sequence[Tuple[int, Optional[str]]], lit: Optional[int] = None):
    """keys ++ aggregates over kernel_cases' columns; filter `i > lit` when lit is given (a literal slot)"""
    b = PlanBuilder()
    used = [n for n, _, _ in kc.SCHEMA if n in set(keys) | {c for _, c in aggs if c} | ({"i"} if lit is not None else set())]
    e = {n: b.col(kc.TYPE[n], kc.COL[n], kc.NULLABLE[n], scale=kc.DEC_SCALE if kc.TYPE[n] == T.DECIMAL else 0) for n in used}
    if lit is not None:
        b.filter(e["i"] > b.lit(T.INT))
    if keys:
        b.group_by(*[e[k] for k in keys])
    for fn, c in aggs:
        b.agg(fn, e[c] if c else None)
    return b.build()


def _value(c: str, v):
    if kc.TYPE[c] == T.FLOAT:
        return float(np.float32(v))
    if kc.TYPE[c] == T.BOOLEAN:
        return bool(v)
    if kc.TYPE[c] == T.DOUBLE:
        return float(v)
    if kc.TYPE[c] in (T.STRING,):
        return bytes(v)
    return int(v)


def _scan(keys, cols, raws, lit):
    """(key tuple, {column: (value, is NULL)}) of every counted row, in scan order"""
    for raw in raws:
        live = raw.live()
        eff = {c: raw.effective(c) for c in set(cols) | set(keys) | ({"i"} if lit is not None else set())}
        for r in range(raw.n):
            if not live[r]:
                continue
            if lit is not None and (eff["i"][1][r] or not eff["i"][0][r] > lit):
                continue
            key = tuple(None if eff[k][1][r] else _value(k, eff[k][0][r]) for k in keys)
            yield key, {c: (None if eff[c][1][r] else _value(c, eff[c][0][r])) for c in cols}


def update_rows(keys, aggs, raws, lit=None) -> List[list]:
    """partial rows by Spark's row-at-a-time update; COUNT(*) counts the rows of the group"""
    cols = sorted({c for _, c in aggs if c})
    groups: Dict[tuple, list] = {}
    for key, vals in _scan(keys, cols, raws, lit):
        bufs = groups.get(key)
        if bufs is None:
            bufs = groups[key] = [0 if fn == AggFn.COUNT_STAR else [None, False] for fn, _ in aggs]
        for j, (fn, c) in enumerate(aggs):
            if fn == AggFn.COUNT_STAR:
                bufs[j] += 1
                continue
            x = vals[c]
            if ignores_nulls(fn) and x is None:
                continue
            b = bufs[j]
            if is_last(fn) or not b[1]:
                b[0] = x
            b[1] = True
    if not keys and not groups:
        groups[()] = [0 if fn == AggFn.COUNT_STAR else [None, False] for fn, _ in aggs]
    return [list(k) + [f for b in bufs for f in (b if isinstance(b, list) else [b])] for k, bufs in groups.items()]


def numpy_rows(keys, aggs, raws, lit=None) -> List[list]:
    """the same partial rows from first / last occurrences found with numpy over the concatenated scan"""
    cols = sorted({c for _, c in aggs if c} | set(keys) | ({"i"} if lit is not None else set()))
    vals = {c: [] for c in cols}
    nuls = {c: [] for c in cols}
    live = []
    for raw in raws:
        for c in cols:
            v, nl = raw.effective(c)
            vals[c] += list(v)
            nuls[c].append(np.asarray(nl, dtype=bool))
        live.append(raw.live())
    nuls = {c: np.concatenate(nuls[c]) if nuls[c] else np.zeros(0, bool) for c in cols}
    keep = np.concatenate(live) if live else np.zeros(0, bool)
    if lit is not None:
        iv = np.array(vals["i"], dtype=np.int64)
        keep = keep & ~nuls["i"] & (iv > lit)
    pos = np.flatnonzero(keep)
    gkeys = [tuple(None if nuls[k][p] else _value(k, vals[k][p]) for k in keys) for p in pos]
    uniq: Dict[tuple, int] = {}
    gid = np.array([uniq.setdefault(k, len(uniq)) for k in gkeys], dtype=np.int64)
    if not keys and not uniq:
        uniq[()] = 0
    ng = len(uniq)
    out = {k: list(k) for k in uniq}
    names = list(uniq)
    for fn, c in aggs:
        if fn == AggFn.COUNT_STAR:
            cnt = np.bincount(gid, minlength=ng)
            for g, k in enumerate(names):
                out[k].append(int(cnt[g]))
            continue
        sel = np.ones(len(pos), bool) if not ignores_nulls(fn) else ~nuls[c][pos]
        idx = np.flatnonzero(sel)
        win = np.full(ng, -1, dtype=np.int64)
        if len(idx):
            order = idx[::-1] if not is_last(fn) else idx   # numpy keeps the last assignment of a repeated index
            win[gid[order]] = order
        for g, k in enumerate(names):
            if win[g] < 0:
                out[k] += [None, False]
            else:
                p = pos[win[g]]
                out[k] += [None if nuls[c][p] else _value(c, vals[c][p]), True]
    return list(out.values())


def merge(fn, left: list, right: list) -> list:
    """Spark's mergeExpressions of [value, valueSet]"""
    if is_last(fn):
        return [right[0] if right[1] else left[0], left[1] or right[1]]
    return [left[0] if left[1] else right[0], left[1] or right[1]]


def canon(v):
    """a field compared exactly: doubles by their bits (NaN payloads, -0.0), everything else by value"""
    if isinstance(v, float):
        return ("f", struct.pack("<d", v))
    if isinstance(v, (bool, np.bool_)):
        return ("i", int(v))
    if isinstance(v, str):
        return ("s", v.encode())
    if isinstance(v, (bytes, bytearray)):
        return ("s", bytes(v))
    if v is None:
        return ("n",)
    return ("i", int(v))


def assert_rows_equal(got: Sequence[list], want: Sequence[list], nkeys: int, what: str = ""):
    g = sorted(([canon(x) for x in r] for r in got), key=lambda r: r[:nkeys])
    w = sorted(([canon(x) for x in r] for r in want), key=lambda r: r[:nkeys])
    assert len(g) == len(w), f"{what}: {len(g)} groups, expected {len(w)}"
    for a, b in zip(g, w):
        assert a == b, f"{what}: group {a[:nkeys]}:\n got      {a}\n expected {b}"


def float_bits(x: float) -> int:
    return struct.unpack("<q", struct.pack("<d", x))[0]


def nan_with_payload(payload: int) -> float:
    return struct.unpack("<d", struct.pack("<q", 0x7FF0000000000000 | (payload & 0x000FFFFFFFFFFFFF) | 1))[0]


def is_nan(x) -> bool:
    return isinstance(x, float) and math.isnan(x)
