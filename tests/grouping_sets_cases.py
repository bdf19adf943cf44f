"""GROUP BY ... WITH ROLLUP / WITH CUBE / GROUPING SETS, engine-agnostic.

Spark 2.1.1 plans these queries as Expand under the partial aggregate (ResolveGroupingAnalytics, restated from upstream Spark:
the fork's analyzer source is not at hand): every row once per grouping set, the keys absent from the set NULL, the set's mask
appended as spark_grouping_id.  `expand_reference` restates that per set: the plain GROUP BY over the set's present keys, its
rows widened with NULLs for the absent keys and the mask -- rows of different sets never meet in one group, so the union of
the per-set results is Expand's result.  A plan with no input rows has no output rows, not even for the () set.

The closed forms are the reference's core/src/test/scala/org/apache/spark/sql/store/CubeRollupGroupingSetsTest.scala:42-90.
"""
import struct
from typing import Callable, List, Sequence

import numpy as np

from snappydata_b200.capi import Op, PlanDesc
from snappydata_b200.column_format import SqlType as T, build_batch, parse_row_stream, unsafe_row
from snappydata_b200.plan import PlanBuilder

MYTABLE = [(1, 2005, 12000), (1, 2006, 18000), (1, 2007, 25000), (2, 2005, 15000), (2, 2006, 6000), (2, 2007, 25000)]

ROLLUP_ROWS = sorted([[1, 2005, 0, 12000], [1, 2006, 0, 18000], [1, 2007, 0, 25000], [2, 2005, 0, 15000], [2, 2006, 0, 6000],
                      [2, 2007, 0, 25000], [1, None, 1, 55000], [2, None, 1, 46000], [None, None, 3, 101000]], key=repr)
CUBE_ROWS = sorted(ROLLUP_ROWS + [[None, 2005, 2, 27000], [None, 2006, 2, 24000], [None, 2007, 2, 50000]], key=repr)


def mytable_batch():
    schema = [("col1", T.INT, True), ("col2", T.INT, True), ("col3", T.INT, True)]
    a = np.array(MYTABLE, dtype=np.int32)
    return build_batch(len(MYTABLE), schema, {"col1": a[:, 0], "col2": a[:, 1], "col3": a[:, 2]}, {})


def mytable_plan(shape: str) -> PlanDesc:
    """SELECT col1, col2, SUM(col3) FROM mytable GROUP BY <shape>"""
    b = PlanBuilder()
    c1, c2, c3 = b.col(T.INT, 0, True), b.col(T.INT, 1, True), b.col(T.INT, 2, True)
    if shape == "rollup":
        b.rollup(c1, c2)
    elif shape == "cube":
        b.cube(c1, c2)
    else:   # GROUPING SETS ((col1, col2), (col1), (col2), ())
        b.grouping_sets([c1, c2], [[c1, c2], [c1], [c2], []])
    b.sum(c3)
    return b.build()


# ---- Expand, restated per set ------------------------------------------------------------------------------------------
def split(desc: PlanDesc):
    """(n GROUP BY key nodes, masks, descriptor without the GROUPING_SET / GROUPING_ID nodes)."""
    gid = desc.keys_py[-1]
    op, _, first, count, _ = desc.exprs_py[gid]
    assert op == Op.GROUPING_ID
    masks = [desc.exprs_py[first + j][2] for j in range(count)]
    assert first + count == gid == len(desc.exprs_py) - 1, "the builder appends the set nodes last"
    return desc.keys_py[:-1], masks, first


def set_plan(desc: PlanDesc, mask: int) -> PlanDesc:
    """the plain GROUP BY over the keys present in the set `mask`"""
    keys, _, first = split(desc)
    n = len(keys)
    present = [k for i, k in enumerate(keys) if not (mask >> (n - 1 - i)) & 1]
    return PlanDesc(desc.cols_py, desc.exprs_py[:first], desc.filter, present, desc.aggs_py, desc.proj_py,
                    desc.literal_types_py)


def widen(desc: PlanDesc, mask: int, rows: Sequence[list]) -> List[list]:
    """rows of set_plan(desc, mask) -> rows of the grouping-sets plan: NULL for the absent keys, then gid"""
    n = len(split(desc)[0])
    out = []
    for r in rows:
        keys, it = [], iter(r)
        for i in range(n):
            keys.append(None if (mask >> (n - 1 - i)) & 1 else next(it))
        out.append(keys + [mask] + list(it))
    return out


def expand_reference(run: Callable, desc: PlanDesc, lits, batches) -> List[list]:
    """final rows of the grouping-sets plan, from one plain GROUP BY per set run by `run(desc, lits, batches) -> (rows, _)`"""
    keys, masks, _ = split(desc)
    finest, _ = run(set_plan(desc, 0), lits, batches)
    if not finest:   # Expand over no rows: no rows, not even for ()
        return []
    out = []
    for m in masks:
        rows, _ = run(set_plan(desc, m), lits, batches)
        out += widen(desc, m, rows)
    return out


def expand_partials(oracle_plan_fn: Callable, desc: PlanDesc, lits, batches) -> bytes:
    """partial rows of the grouping-sets plan, built from the oracle's partial rows of each set's plain plan (row stream
    [int64 size][UnsafeRow(keys, gid, buffers)])"""
    _, masks, _ = split(desc)
    schema = desc.partial_schema()
    out = bytearray()
    for m in masks:
        sp = set_plan(desc, m)
        raw = oracle_plan_fn(sp, lits, batches)
        for r in widen(desc, m, parse_row_stream(raw, sp.partial_schema())):
            row = unsafe_row(list(zip(schema, r)))
            out += struct.pack("<q", len(row)) + row
    return bytes(out)


def by_gid(rows: Sequence[list], gid_index: int):
    out = {}
    for r in rows:
        out.setdefault(r[gid_index], []).append(r)
    return out


# ---- closed forms of CubeRollupGroupingSetsTest -----------------------------------------------------------------------
def case_rollup_closed_form(run):
    rows, _ = run(mytable_plan("rollup"), [], [mytable_batch()])
    assert sorted(rows, key=repr) == ROLLUP_ROWS


def case_cube_closed_form(run):
    rows, _ = run(mytable_plan("cube"), [], [mytable_batch()])
    assert sorted(rows, key=repr) == CUBE_ROWS


def case_grouping_sets_closed_form(run):
    rows, _ = run(mytable_plan("sets"), [], [mytable_batch()])
    assert sorted(rows, key=repr) == CUBE_ROWS


CLOSED_FORMS = [case_rollup_closed_form, case_cube_closed_form, case_grouping_sets_closed_form]
