"""Plan construction: a small expression DSL that flattens to ``sd_plan_desc`` (include/snappy_gpu.h),
standing in for what the Scala operators would serialise from the Catalyst trees of
FilterExec / ProjectExec / the aggregate functions (SURVEY.md 8a a12-a16).

Literals are *slots* whose values are supplied per execution (``Plan.set_literals``), mirroring
the reference's ParamLiteral tokenisation (core/catalyst/expressions/ParamLiteral.scala:43-110):
one compiled plan serves every literal value.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

from .capi import SD_PLAN_MUTATE, AggFn, Op, PlanDesc
from .column_format import SqlType

_NUMERIC_RANK = {SqlType.BYTE: 1, SqlType.SHORT: 2, SqlType.INT: 3, SqlType.LONG: 4, SqlType.FLOAT: 5, SqlType.DOUBLE: 6}


class E:
    """Expression node under construction."""

    def __init__(self, b: "PlanBuilder", op: int, t: SqlType, a: object = 0, bb: object = 0, c: int = 0):
        self.b, self.op, self.t, self.a, self.bb, self.c = b, op, SqlType(t), a, bb, c   # DECIMAL LIT / CAST: c = (precision << 8) | scale

    # -- arithmetic (operands must already have the same type; use cast()) ---------------------
    def _bin(self, op, other, t=None):
        other = self.b.coerce(other, self.t)
        return E(self.b, op, t or self.t, self, other)

    def __add__(self, o): return self._bin(Op.ADD, o)
    def __sub__(self, o): return self._bin(Op.SUB, o)
    def __mul__(self, o): return self._bin(Op.MUL, o)
    def __truediv__(self, o): return self._bin(Op.DIV, o)
    def __radd__(self, o): return self.b.coerce(o, self.t)._bin(Op.ADD, self)
    def __rsub__(self, o): return self.b.coerce(o, self.t)._bin(Op.SUB, self)
    def __rmul__(self, o): return self.b.coerce(o, self.t)._bin(Op.MUL, self)
    def __neg__(self): return E(self.b, Op.NEG, self.t, self)

    # -- comparisons -> BOOLEAN ---------------------------------------------------------------
    def __lt__(self, o): return self._bin(Op.LT, o, SqlType.BOOLEAN)
    def __le__(self, o): return self._bin(Op.LE, o, SqlType.BOOLEAN)
    def __gt__(self, o): return self._bin(Op.GT, o, SqlType.BOOLEAN)
    def __ge__(self, o): return self._bin(Op.GE, o, SqlType.BOOLEAN)
    def eq(self, o): return self._bin(Op.EQ, o, SqlType.BOOLEAN)
    def ne(self, o): return self._bin(Op.NE, o, SqlType.BOOLEAN)

    def __and__(self, o): return E(self.b, Op.AND, SqlType.BOOLEAN, self, o)
    def __or__(self, o): return E(self.b, Op.OR, SqlType.BOOLEAN, self, o)
    def __invert__(self): return E(self.b, Op.NOT, SqlType.BOOLEAN, self)

    def is_null(self): return E(self.b, Op.ISNULL, SqlType.BOOLEAN, self)
    def is_not_null(self): return E(self.b, Op.ISNOTNULL, SqlType.BOOLEAN, self)
    def cast(self, t: SqlType, precision: int = 0, scale: int = 0):
        if SqlType(t) == self.t and SqlType(t) != SqlType.DECIMAL:
            return self
        return E(self.b, Op.CAST, t, self, 0, (precision << 8) | scale if SqlType(t) == SqlType.DECIMAL else 0)
    def startswith(self, lit: "E"): return E(self.b, Op.STARTSWITH, SqlType.BOOLEAN, self, lit)

    def isin(self, n: int):
        """IN over ``n`` fresh literal slots of this expression's type."""
        first = len(self.b.literal_types)
        for _ in range(n):
            self.b.literal_types.append(self.t)
        return E(self.b, Op.IN, SqlType.BOOLEAN, self, first, n)


class PlanBuilder:
    def __init__(self):
        self.cols: List[Tuple[SqlType, bool, int, int]] = []
        self.literal_types: List[SqlType] = []
        self._filter: Optional[E] = None
        self._keys: List[E] = []
        self._sets: Optional[List[int]] = None   # grouping-set masks (rollup / cube / grouping_sets)
        self._aggs: List[Tuple[int, Optional[E]]] = []
        self._proj: List[E] = []
        self._flags = 0
        self._targets: List[int] = []

    # scan columns (ColumnTableScan.output)
    def col(self, t: SqlType, table_ordinal: int, nullable: bool = False, scale: int = 0, precision: int = 0) -> E:
        if SqlType(t) == SqlType.DECIMAL and not precision:
            precision = 18
        self.cols.append((SqlType(t), bool(nullable), int(table_ordinal), int(scale), int(precision)))
        return E(self, Op.COL, t, len(self.cols) - 1)

    def lit(self, t: SqlType, precision: int = 0, scale: int = 0) -> E:
        """A runtime literal slot (a DECIMAL literal's value is its unscaled integer at `scale`)."""
        self.literal_types.append(SqlType(t))
        return E(self, Op.LIT, t, len(self.literal_types) - 1, 0, (precision << 8) | scale if SqlType(t) == SqlType.DECIMAL else 0)

    def coerce(self, x, t: SqlType) -> E:
        if isinstance(x, E):
            return x
        raise TypeError("constants must be literal slots: use PlanBuilder.lit(type) and pass the value "
                        "with Plan.set_literals (the reference tokenises constants the same way)")

    def filter(self, e: E): self._filter = e; return self
    def group_by(self, *keys: E): self._keys = list(keys); self._sets = None; return self

    # GROUP BY ... WITH ROLLUP / WITH CUBE / GROUPING SETS: the keys, then spark_grouping_id (an INT key whose value is the set's
    # mask; bit (n-1-k) set <=> key k is absent, SnappyParser.extractGroupingSet)
    def grouping_sets(self, keys: Sequence[E], sets: Sequence[Sequence[E]]):
        """GROUPING SETS: each set is a list of some of `keys` (the others are NULL in its rows)."""
        keys = list(keys)
        n = len(keys)
        masks = []
        for st in sets:
            present = {id(e) for e in st}
            unknown = [e for e in st if all(e is not k for k in keys)]
            if unknown:
                raise ValueError("a grouping set may only name GROUP BY expressions")
            masks.append(sum(1 << (n - 1 - k) for k, e in enumerate(keys) if id(e) not in present))
        return self.grouping_masks(keys, masks)

    def grouping_masks(self, keys: Sequence[E], masks: Sequence[int]):
        self._keys = list(keys)
        self._sets = [int(m) for m in masks]
        return self

    def rollup(self, *keys: E):
        n = len(keys)
        return self.grouping_masks(keys, [(1 << i) - 1 for i in range(n + 1)])

    def cube(self, *keys: E):
        return self.grouping_masks(keys, list(range(1 << len(keys))))

    def agg(self, fn: int, e: Optional[E] = None): self._aggs.append((fn, e)); return self
    def sum(self, e: E): return self.agg(AggFn.SUM, e)
    def avg(self, e: E): return self.agg(AggFn.AVG, e)
    def min(self, e: E): return self.agg(AggFn.MIN, e)
    def max(self, e: E): return self.agg(AggFn.MAX, e)
    def count(self, e: Optional[E] = None): return self.agg(AggFn.COUNT if e is not None else AggFn.COUNT_STAR, e)
    # moment aggregates take a DOUBLE input, as Spark casts it (ImplicitCastInputTypes): e.cast(SqlType.DOUBLE)
    def stddev_pop(self, e: E): return self.agg(AggFn.STDDEV_POP, e)
    def stddev_samp(self, e: E): return self.agg(AggFn.STDDEV_SAMP, e)
    def var_pop(self, e: E): return self.agg(AggFn.VAR_POP, e)
    def var_samp(self, e: E): return self.agg(AggFn.VAR_SAMP, e)
    def skewness(self, e: E): return self.agg(AggFn.SKEWNESS, e)
    def kurtosis(self, e: E): return self.agg(AggFn.KURTOSIS, e)
    stddev, variance = stddev_samp, var_samp
    # two-input aggregates over a PAIR node of DOUBLE inputs (Spark casts them too): x.cast(SqlType.DOUBLE)
    def pair(self, x: E, y: E) -> E: return E(self, Op.PAIR, SqlType.DOUBLE, x, y)
    def covar_pop(self, x: E, y: E): return self.agg(AggFn.COVAR_POP, self.pair(x, y))
    def covar_samp(self, x: E, y: E): return self.agg(AggFn.COVAR_SAMP, self.pair(x, y))
    def corr(self, x: E, y: E): return self.agg(AggFn.CORR, self.pair(x, y))
    # Spark's first / first_value and last / last_value: the value of the first / last row in scan order
    def first(self, e: E, ignore_nulls: bool = False): return self.agg(AggFn.FIRST_IGNORE_NULLS if ignore_nulls else AggFn.FIRST, e)
    def last(self, e: E, ignore_nulls: bool = False): return self.agg(AggFn.LAST_IGNORE_NULLS if ignore_nulls else AggFn.LAST, e)
    def project(self, *es: E): self._proj = list(es); return self

    # UPDATE / DELETE over a resident store (SD_PLAN_MUTATE; the WHERE clause is filter())
    def update(self, assignments: Dict[int, E]):
        """UPDATE ... SET table column k = assignments[k], ...: the values become the plan's projection."""
        self._targets = [int(k) for k in assignments]
        self._proj = [assignments[k] for k in assignments]
        self._flags = SD_PLAN_MUTATE
        return self

    def delete(self):
        self._targets, self._proj, self._flags = [], [], SD_PLAN_MUTATE
        return self

    def build(self) -> PlanDesc:
        nodes: List[Tuple[int, int, int, int, int]] = []
        memo = {}

        def emit(e: E) -> int:
            if id(e) in memo:
                return memo[id(e)]
            if e.op in (Op.COL, Op.LIT):
                rec = (e.op, int(e.t), int(e.a), 0, int(e.c))
            elif e.op == Op.IN:
                rec = (e.op, int(e.t), emit(e.a), int(e.bb), int(e.c))
            elif e.op in (Op.NEG, Op.CAST, Op.NOT, Op.ISNULL, Op.ISNOTNULL):
                rec = (e.op, int(e.t), emit(e.a), 0, int(e.c) if e.op == Op.CAST else 0)
            else:
                ia = emit(e.a)
                ib = emit(e.bb)
                rec = (e.op, int(e.t), ia, ib, 0)
            nodes.append(rec)
            memo[id(e)] = len(nodes) - 1
            return memo[id(e)]

        f = emit(self._filter) if self._filter is not None else -1
        keys = [emit(k) for k in self._keys]
        aggs = [(fn, emit(e) if e is not None else -1) for fn, e in self._aggs]
        proj = [emit(p) for p in self._proj]
        if self._sets is not None:   # appended last: the scan's generated source is the plain GROUP BY's
            first = len(nodes)
            nodes.extend((Op.GROUPING_SET, int(SqlType.INT), m, 0, 0) for m in self._sets)
            nodes.append((Op.GROUPING_ID, int(SqlType.INT), first, len(self._sets), 0))
            keys.append(len(nodes) - 1)
        return PlanDesc(self.cols, nodes, f, keys, aggs, proj, self.literal_types, self._flags, self._targets)


# ---- the benchmark plans ------------------------------------------------------------------------
# lineitem table columns (cluster/src/test/scala/io/snappydata/benchmark/TPCHTableSchema.scala:122-143)
LINEITEM_COLUMNS = ["l_orderkey", "l_partkey", "l_suppkey", "l_linenumber", "l_quantity", "l_extendedprice",
                    "l_discount", "l_tax", "l_returnflag", "l_linestatus", "l_shipdate", "l_commitdate",
                    "l_receiptdate", "l_shipinstruct", "l_shipmode", "l_comment"]
L_QUANTITY, L_EXTENDEDPRICE, L_DISCOUNT, L_TAX, L_RETURNFLAG, L_LINESTATUS, L_SHIPDATE = 4, 5, 6, 7, 8, 9, 10


def q6_plan() -> PlanDesc:
    """TPC-H Q6 as planned by the reference (TPCH_Queries.scala:600-613):
    ColumnTableScan[l_shipdate,l_discount,l_quantity,l_extendedprice] -> FilterExec -> partial
    SnappyHashAggregateExec(no keys, sum(l_extendedprice * l_discount)).
    Literal slots: 0 d0 (DATE), 1 d1 (DATE), 2 lo (DOUBLE), 3 hi (DOUBLE), 4 quantity (DOUBLE); the
    driver folds `0.06 - 0.01` etc. in DECIMAL before they reach the plan (SURVEY.md Appendix B.7)."""
    b = PlanBuilder()
    ship = b.col(SqlType.DATE, L_SHIPDATE)
    disc = b.col(SqlType.DOUBLE, L_DISCOUNT)
    qty = b.col(SqlType.DOUBLE, L_QUANTITY)
    price = b.col(SqlType.DOUBLE, L_EXTENDEDPRICE)
    d0, d1 = b.lit(SqlType.DATE), b.lit(SqlType.DATE)
    lo, hi, q = b.lit(SqlType.DOUBLE), b.lit(SqlType.DOUBLE), b.lit(SqlType.DOUBLE)
    b.filter((ship >= d0) & (ship < d1) & (disc >= lo) & (disc <= hi) & (qty < q))
    b.sum(price * disc)
    return b.build()


Q6_LITERALS = [8766, 9131, 0.05, 0.07, 24.0]   # 1994-01-01, 1995-01-01, 0.06 -/+ 0.01 folded in DECIMAL, 24


def q1_plan() -> PlanDesc:
    """TPC-H Q1 (TPCH_Queries.scala:125-149): scan 7 columns, filter l_shipdate <= cutoff, group by
    (l_returnflag, l_linestatus), 8 aggregates = 11 buffer fields.
    Literal slots: 0 cutoff (DATE), 1 and 2 the constant 1 (DOUBLE) of (1-l_discount), (1+l_tax)."""
    b = PlanBuilder()
    qty = b.col(SqlType.DOUBLE, L_QUANTITY)
    price = b.col(SqlType.DOUBLE, L_EXTENDEDPRICE)
    disc = b.col(SqlType.DOUBLE, L_DISCOUNT)
    tax = b.col(SqlType.DOUBLE, L_TAX)
    rf = b.col(SqlType.STRING, L_RETURNFLAG)
    ls = b.col(SqlType.STRING, L_LINESTATUS)
    ship = b.col(SqlType.DATE, L_SHIPDATE)
    cutoff = b.lit(SqlType.DATE)
    one_a, one_b = b.lit(SqlType.DOUBLE), b.lit(SqlType.DOUBLE)
    b.filter(ship <= cutoff)
    b.group_by(rf, ls)
    disc_price = price * (one_a - disc)
    b.sum(qty).sum(price).sum(disc_price).sum(disc_price * (one_b + tax))
    b.avg(qty).avg(price).avg(disc).count()
    return b.build()


Q1_LITERALS = [10136, 1.0, 1.0]   # DATE_SUB('1997-12-31', 90) = 1997-10-02


def c1_plan() -> PlanDesc:
    """BASELINE.json configs[0]: SELECT COUNT(*) FROM t WHERE c1 > k over one INT NOT NULL column."""
    b = PlanBuilder()
    c1 = b.col(SqlType.INT, 0)
    b.filter(c1 > b.lit(SqlType.INT))
    b.count()
    return b.build()


# plans compiled ahead of time into libsnappygpu.so (every other plan goes through NVRTC at plan time)
AOT_PLANS = {"c1": c1_plan, "q6": q6_plan, "q1": q1_plan}
