"""Scenarios whose aggregates are exact by construction, and a plain Python evaluator of them.

The scan kernel picks its code per batch (staged vector loads, loads plus NULL prefixes, loads plus delta / delete
patches, or the general per-row decode) and its group table per launch.  To see one wrong row on any of those paths
the results must be compared exactly, so the data is built such that every aggregate has one right answer whatever the
summation order:

  * DOUBLE values are k/16 with |k| < 2^24 and FLOAT values k/16 with |k| < 2^20: every partial sum of up to 2^20 rows
    is a representable double, so SUM / AVG come back bit for bit;
  * INT / LONG are plain integers; LONG values sit near 2^62 so that their sum wraps (Java `long`, as Spark 2.1.1 adds);
  * DECIMAL(18, 2) values span +-(10^18 - 1): the low 32-bit halves the kernel sums separately carry many times;
  * special doubles live in their own groups, chosen by the group's number: NaN, +inf, -inf, +inf with -inf, only
    +-0.0, only NULL;
  * STRING keys and MIN / MAX inputs include bytes >= 0x80, the empty string and strings that prefix each other.

`evaluate` computes the partial rows (keys ++ aggregate buffers, the layout sd_plan_finish emits) from the raw values:
effective value = depth-0 delta, else depth-1 delta, else base; deleted rows dropped; then the filter, the groups and
COUNT(*) / COUNT / SUM / AVG / MIN / MAX with Python integers and exact sums.  It never calls the C oracle:
tests/test_exact_reference.py checks it against the oracle, tests/test_gpu_kernel_paths.py checks the kernel against it.
"""
import math
import struct
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from snappydata_b200.capi import AggFn
from snappydata_b200.column_format import ColumnBatch, SqlType as T, build_batch, encode_delete, encode_delta
from snappydata_b200.plan import PlanBuilder

# table columns: (name, type, nullable)
SCHEMA = [("k", T.STRING, True), ("i", T.INT, True), ("l", T.LONG, False), ("f", T.FLOAT, True), ("d", T.DOUBLE, True),
          ("m", T.DECIMAL, True), ("s", T.STRING, True), ("b", T.BOOLEAN, True), ("t", T.TIMESTAMP, True),
          ("sh", T.SHORT, True), ("dt", T.DATE, True), ("h", T.INT, False)]
COL = {name: i for i, (name, _, _) in enumerate(SCHEMA)}
TYPE = {name: t for name, t, _ in SCHEMA}
NULLABLE = {name: n for name, _, n in SCHEMA}
DEC_SCALE = 2
DEC_MAX = 10 ** 18 - 1
LONG_BASE = 1 << 62

# STRING MIN / MAX inputs: unsigned byte order, prefixes, the empty string, bytes >= 0x80 (no NUL: the dictionary
# writer keeps values in numpy 'S' arrays, which drop trailing NULs)
STRINGS = [b"", b"a", b"ab", b"abc", b"A", b"zz", b"\x7f", b"\x80", b"\x80\x80", b"ab\x80", b"\xc3\xa9", b"\xfe\xff", b"\xff"]
DELTA_ONLY_KEY = b"\xe2\x82\xac-delta-only"   # a key value that exists only in update deltas

# batch kinds -> the decode path the engine should pick for them
KINDS = ("all_fast", "fast_nulls", "fast_overlay", "rle", "dictionary", "bigdictionary", "bitset")
KIND_PATH = {"all_fast": "all_fast", "fast_nulls": "fast_nulls", "fast_overlay": "fast_overlay", "rle": "general",
             "dictionary": "general", "bigdictionary": "general", "bitset": "general"}
ENCODERS = {
    "all_fast": {"b": "uncompressed"},
    "fast_nulls": {"b": "uncompressed"},
    "fast_overlay": {"b": "uncompressed"},
    "rle": {"k": "rle", "i": "rle", "l": "rle", "t": "rle", "sh": "rle", "dt": "rle", "b": "uncompressed"},
    "dictionary": {"i": "dictionary", "l": "dictionary", "t": "dictionary", "dt": "dictionary", "b": "uncompressed"},
    "bigdictionary": {"k": "bigdictionary", "s": "bigdictionary", "i": "bigdictionary", "t": "bigdictionary",
                      "b": "uncompressed"},
    "bitset": {"b": "bitset"},
}
# batch sizes around the 1024-row tile, the 2048-row work item (SD_TUNE_CHUNK_ROWS=2048) and a 20 k-row batch
BOUNDARY_SIZES = (1, 31, 33, 511, 513, 1023, 1024, 1025, 2047, 2049, 3 * 2048 + 77, 20000)


def key_of(g: int) -> bytes:
    """Group g's key: ASCII for even g, a multi-byte UTF-8 prefix (bytes >= 0x80) for odd g."""
    return (b"g%05d" % g) if g % 2 == 0 else (b"\xe2\x82\xac%d" % g)


def hash_key_of(g: int) -> int:
    return g * 7919 - 500000000


@dataclass
class RawBatch:
    """The values behind one ColumnBatch: base values + NULL masks, update deltas, deleted positions."""
    n: int
    values: Dict[str, np.ndarray]
    nulls: Dict[str, np.ndarray]
    deltas: List[Tuple[int, str, np.ndarray, np.ndarray, Optional[np.ndarray]]] = field(default_factory=list)
    deletes: np.ndarray = field(default_factory=lambda: np.zeros(0, dtype=np.int32))

    def effective(self, name: str) -> Tuple[list, np.ndarray]:
        """(values as a Python list, NULL mask) after the deltas: depth 0 wins over depth 1, which wins over the base."""
        vals = list(self.values[name].tolist())
        nul = self.nulls.get(name, np.zeros(self.n, dtype=bool)).copy()
        for depth in (1, 0):
            for d, col, pos, v, dn in self.deltas:
                if d != depth or col != name:
                    continue
                vl = v.tolist()
                for j, p in enumerate(pos.tolist()):
                    vals[p] = vl[j]
                    nul[p] = bool(dn[j]) if dn is not None else False
        return vals, nul

    def live(self) -> np.ndarray:
        m = np.ones(self.n, dtype=bool)
        m[self.deletes] = False
        return m


def boundary_rows(n: int) -> np.ndarray:
    """Rows where tiles (1024 rows at 4 rows per thread), work items (2048 / 8192 / 16384 rows) and null words start / end."""
    b = {0, 1, 31, 32, 63, 64, 511, 512, 1023, 1024, 1025, 2047, 2048, 2049, 4095, 4096, 6143, 6144, 8191, 8192, 16383,
         16384, n - 2, n - 1}
    return np.array(sorted(x for x in b if 0 <= x < n), dtype=np.int32)


def _runs(n: int, rng) -> np.ndarray:
    """Run id per row: runs of 1..40 rows, plus runs that straddle the tile / work-item boundaries 1024 and 2048."""
    starts = [0]
    while starts[-1] < n:
        starts.append(starts[-1] + int(rng.integers(1, 41)))
    starts = set(s for s in starts if s < n)
    for lo, hi in ((1000, 1100), (2040, 2060), (8180, 8200)):
        starts = {s for s in starts if not lo < s < hi}
        if lo < n:
            starts.add(lo)
    starts = np.array(sorted(starts))
    run = np.zeros(n, dtype=np.int64)
    run[starts[1:]] = 1
    return np.cumsum(run)


def _doubles(rng, m: int, bits: int) -> np.ndarray:
    return rng.integers(-(2 ** bits - 1), 2 ** bits, m).astype(np.float64) / 16.0


def make_batch(n: int, kind: str, seed: int, groups: int, batch_id: int = 0, group_base: int = 0,
               distinct_groups: bool = False) -> Tuple[ColumnBatch, RawBatch]:
    """One batch of `kind` (KINDS).  Keys are drawn from groups [group_base, group_base + groups) (every row its own
    group in order when `distinct_groups`)."""
    rng = np.random.default_rng(seed)
    nulls_ok = kind not in ("all_fast", "fast_overlay")
    mutated = kind not in ("all_fast", "fast_nulls")
    run = _runs(n, rng)
    nruns = int(run[-1]) + 1 if n else 0

    def per_run(v):
        return v[run]

    if distinct_groups:
        g = group_base + np.arange(n)
    else:
        g = per_run(group_base + rng.integers(0, groups, nruns))
    cls = g % 8
    vals: Dict[str, np.ndarray] = {}
    vals["k"] = np.array([key_of(int(x)) for x in g], dtype=object)
    vals["h"] = np.array([hash_key_of(int(x)) for x in g], dtype=np.int64).astype(np.int32)
    vals["i"] = per_run(rng.integers(-1000, 1000, nruns)).astype(np.int32)
    vals["l"] = per_run(LONG_BASE + rng.integers(-1000, 1000, nruns)).astype(np.int64)
    vals["t"] = per_run(rng.integers(-10 ** 15, 10 ** 15, nruns)).astype(np.int64)
    vals["sh"] = per_run(rng.integers(-32768, 32768, nruns)).astype(np.int16)
    vals["dt"] = per_run(rng.integers(-20000, 40000, nruns)).astype(np.int32)
    vals["f"] = (rng.integers(-(2 ** 20 - 1), 2 ** 20, n).astype(np.float64) / 16.0).astype(np.float32)
    d = _doubles(rng, n, 24)
    r = rng.random(n)
    d[(cls == 1) & (r < 0.05)] = np.nan
    d[(cls == 2) & (r < 0.05)] = np.inf
    d[(cls == 3) & (r < 0.03)] = np.inf
    d[(cls == 3) & (r > 0.97)] = -np.inf
    d[cls == 4] = np.where(r[cls == 4] < 0.5, 0.0, -0.0)
    d[(cls == 6) & (r < 0.05)] = -np.inf
    vals["d"] = d
    f = vals["f"]
    f[(cls == 1) & (r < 0.05)] = np.nan
    f[cls == 4] = np.where(r[cls == 4] < 0.5, 0.0, -0.0).astype(np.float32)
    vals["m"] = rng.integers(-DEC_MAX, DEC_MAX + 1, n, dtype=np.int64)
    vals["s"] = np.array([STRINGS[x] for x in rng.integers(0, len(STRINGS), n)], dtype=object)
    vals["b"] = rng.random(n) < 0.5

    nulls: Dict[str, np.ndarray] = {}
    for name, _, nullable in SCHEMA:
        if nullable:
            nulls[name] = np.zeros(n, dtype=bool)
    if nulls_ok:
        for name in nulls:
            nulls[name] |= rng.random(n) < 0.08
        nulls["d"] |= cls == 5                         # groups whose DOUBLE input is all NULL
        nulls["f"] |= cls == 5
        nulls["m"][:32] = True                         # a NULL run on the first null word
        nulls["s"][max(0, n - 33):] = True             # ... and on the last one
        if n >= 2048:                                  # a whole 1024-row tile of NULLs
            for name in ("i", "d", "f"):
                nulls[name][1024:2048] = True
        nulls["k"][boundary_rows(n)[::3]] = True       # NULL keys on boundary rows

    raw = RawBatch(n, vals, nulls)
    if mutated and n:
        bnd = boundary_rows(n)
        p1 = np.unique(np.concatenate([bnd, rng.choice(n, size=min(n, 60), replace=False)])).astype(np.int32)
        p0 = np.unique(np.concatenate([bnd[::2], rng.choice(n, size=min(n, 40), replace=False)])).astype(np.int32)
        for depth, pos in ((0, p0), (1, p1)):
            m = len(pos)
            for name in ("i", "l", "d", "k"):
                if name == "i":
                    v = rng.integers(-1000, 1000, m).astype(np.int32)
                elif name == "l":
                    v = (LONG_BASE + rng.integers(-1000, 1000, m)).astype(np.int64)
                elif name == "d":
                    v = _doubles(rng, m, 24)
                else:
                    v = np.array([key_of(int(x)) for x in group_base + rng.integers(0, groups, m)], dtype=object)
                    v[: max(1, m // 8)] = DELTA_ONLY_KEY
                dn = (rng.random(m) < 0.25) if NULLABLE[name] else None
                raw.deltas.append((depth, name, pos, v, dn))
        dels = set(boundary_rows(n).tolist()) | set(rng.choice(n, size=max(1, n // 40), replace=False).tolist())
        if n >= 8192:
            dels |= set(range(2048, 4096))             # a whole 2048-row work item deleted
        if len(dels) >= n:
            dels.discard(n - 1)
        raw.deletes = np.array(sorted(dels), dtype=np.int32)

    batch = build_batch(n, SCHEMA, vals, nulls, batch_id=batch_id, bucket_id=batch_id % 4, encoders=ENCODERS[kind])
    batch.stats = None      # no batch skipping: every batch reaches the kernel
    for depth, name, pos, v, dn in raw.deltas:
        (batch.delta0 if depth == 0 else batch.delta1)[COL[name]] = encode_delta(n, pos, v, TYPE[name], dn)
    if len(raw.deletes):
        batch.delete_mask = encode_delete(n, raw.deletes)
    return batch, raw


# ---- queries --------------------------------------------------------------------------------------------------------
@dataclass
class Query:
    """keys, aggregates ((AggFn, column name or None)), and an optional filter `i IS NULL OR i > lit`."""
    keys: Sequence[str]
    aggs: Sequence[Tuple[int, Optional[str]]]
    filter_lit: Optional[int] = None

    def columns(self) -> List[str]:
        used = set(self.keys) | {c for _, c in self.aggs if c} | ({"i"} if self.filter_lit is not None else set())
        return [name for name, _, _ in SCHEMA if name in used]

    def desc(self):
        b = PlanBuilder()
        e = {name: b.col(TYPE[name], COL[name], NULLABLE[name], scale=DEC_SCALE if TYPE[name] == T.DECIMAL else 0)
             for name in self.columns()}
        if self.filter_lit is not None:
            b.filter(e["i"].is_null() | (e["i"] > b.lit(T.INT)))
        if self.keys:
            b.group_by(*[e[k] for k in self.keys])
        for fn, c in self.aggs:
            b.agg(fn, e[c] if c else None)
        return b.build()

    def literals(self) -> list:
        return [] if self.filter_lit is None else [self.filter_lit]

    def field_kinds(self) -> List[str]:
        """Kind of every partial-row field: key / count / sum / avg_sum / avg_count / min / max."""
        out = ["key"] * len(self.keys)
        for fn, _ in self.aggs:
            out += {AggFn.COUNT_STAR: ["count"], AggFn.COUNT: ["count"], AggFn.SUM: ["sum"], AggFn.AVG: ["avg_sum", "avg_count"],
                    AggFn.MIN: ["min"], AggFn.MAX: ["max"]}[fn]
        return out


EVERY_AGG = [(AggFn.COUNT_STAR, None), (AggFn.COUNT, "i"), (AggFn.SUM, "i"), (AggFn.SUM, "l"), (AggFn.SUM, "f"),
             (AggFn.SUM, "d"), (AggFn.SUM, "m"), (AggFn.AVG, "i"), (AggFn.AVG, "d"), (AggFn.AVG, "m"), (AggFn.AVG, "f"),
             (AggFn.MIN, "d"), (AggFn.MAX, "d"), (AggFn.MIN, "f"), (AggFn.MAX, "f"), (AggFn.MIN, "s"), (AggFn.MAX, "s"),
             (AggFn.MIN, "i"), (AggFn.MAX, "l"), (AggFn.MIN, "m"), (AggFn.MAX, "m"), (AggFn.MIN, "t"), (AggFn.MAX, "dt"),
             (AggFn.SUM, "sh"), (AggFn.COUNT, "b")]


# ---- the evaluator --------------------------------------------------------------------------------------------------
def _wrap64(x: int) -> int:
    return ((x + (1 << 63)) % (1 << 64)) - (1 << 63)


def _exact_sum(xs: Sequence[float]) -> float:
    """Sum of k/16 values (and specials): exact rational sum, checked against math.fsum."""
    if any(math.isnan(x) for x in xs) or (math.inf in xs and -math.inf in xs):
        return math.nan
    if math.inf in xs:
        return math.inf
    if -math.inf in xs:
        return -math.inf
    sixteenths = 0
    for x in xs:
        k = x * 16.0
        assert k == int(k), f"{x!r} is not a multiple of 1/16: the scenario is not exact"
        sixteenths += int(k)
    s = sixteenths / 16.0
    assert s * 16.0 == sixteenths, "sum not representable"
    assert math.fsum(xs) == s
    return s + 0.0          # an exact zero is +0.0, as an accumulator that starts at +0.0 leaves it


def _nan_safe_key(x: float):
    """Spark's nanSafeCompare order: NaN greatest, -0.0 == 0.0."""
    return (1, 0.0) if math.isnan(x) else (0, x + 0.0)


def _min_max(fn: int, xs: list, t: T):
    if not xs:
        return None
    if t in (T.FLOAT, T.DOUBLE):
        pick = min(xs, key=_nan_safe_key) if fn == AggFn.MIN else max(xs, key=_nan_safe_key)
        return float(np.float32(pick)) if t == T.FLOAT else pick
    return min(xs) if fn == AggFn.MIN else max(xs)


def evaluate(query: Query, raws: Sequence[RawBatch]) -> List[list]:
    """Partial rows of `query` over the batches (group order unspecified)."""
    cols = set(query.columns())
    keys_all: List[tuple] = []
    vals_all: Dict[str, list] = {c: [] for c in cols}
    nul_all: Dict[str, list] = {c: [] for c in cols}
    for raw in raws:
        live = raw.live()
        eff = {c: raw.effective(c) for c in cols}
        keep = live.copy()
        if query.filter_lit is not None:
            iv, inul = eff["i"]
            keep &= np.array([bool(inul[j]) or iv[j] > query.filter_lit for j in range(raw.n)], dtype=bool)
        rows = np.flatnonzero(keep).tolist()
        for c in cols:
            v, nl = eff[c]
            vals_all[c] += [v[j] for j in rows]
            nul_all[c] += [bool(nl[j]) for j in rows]
        keys_all += [tuple(None if eff[k][1][j] else eff[k][0][j] for k in query.keys) for j in rows]
    groups: Dict[tuple, List[int]] = {}
    for j, key in enumerate(keys_all):
        groups.setdefault(key, []).append(j)
    if not query.keys:
        groups = {(): list(range(len(keys_all)))}
    out = []
    for key, idx in groups.items():
        row = list(key)
        for fn, c in query.aggs:
            if fn == AggFn.COUNT_STAR:
                row.append(len(idx))
                continue
            t = TYPE[c]
            xs = [vals_all[c][j] for j in idx if not nul_all[c][j]]
            if t == T.FLOAT:
                xs = [float(np.float32(x)) for x in xs]
            if fn == AggFn.COUNT:
                row.append(len(xs))
            elif fn == AggFn.SUM:
                if not xs:
                    row.append(None)
                elif t in (T.FLOAT, T.DOUBLE):
                    row.append(_exact_sum(xs))
                elif t == T.DECIMAL:
                    row.append(sum(int(x) for x in xs))
                else:
                    row.append(_wrap64(sum(int(x) for x in xs)))
            elif fn == AggFn.AVG:
                if t == T.DECIMAL:
                    row += [sum(int(x) for x in xs), len(xs)]
                else:
                    row += [_exact_sum([float(x) for x in xs]) if xs else 0.0, len(xs)]
            else:
                row.append(_min_max(fn, xs, t))
        out.append(row)
    return out


def decimal_avg_half_up(unscaled_sum: int, count: int) -> Optional[int]:
    """AVG over DECIMAL(p, s): sum / count at scale s + 4, rounded HALF_UP (java.math.BigDecimal) -> unscaled."""
    if count == 0:
        return None
    q, r = divmod(abs(unscaled_sum) * 10 ** 4, count)
    if 2 * r >= count:
        q += 1
    return -q if unscaled_sum < 0 else q


def final_rows(query: Query, partial: Sequence[list]) -> List[list]:
    """The final aggregate values from the partial rows (AVG = sum / count; DECIMAL AVG rounded HALF_UP)."""
    out = []
    for r in partial:
        row, j = list(r[: len(query.keys)]), len(query.keys)
        for fn, c in query.aggs:
            if fn == AggFn.AVG:
                s, n = r[j], r[j + 1]
                row.append(decimal_avg_half_up(s, n) if TYPE[c] == T.DECIMAL else (s / n if n else None))
                j += 2
            else:
                row.append(r[j])
                j += 1
        out.append(row)
    return out


# ---- exact comparison -----------------------------------------------------------------------------------------------
def _sort_key(r, nkeys):
    return tuple((0, b"") if v is None else (1, v) if isinstance(v, bytes) else (2, v) for v in r[:nkeys])


def _bits(x: float) -> bytes:
    return struct.pack("<d", x)


def assert_rows_exact(got: Sequence[list], want: Sequence[list], query: Query, what: str = ""):
    """Every field equal: integers / DECIMAL / strings / counts exactly, doubles bit for bit, NaN as NaN; MIN / MAX whose
    answer is +-0.0 as values (which zero wins a tie is order-dependent: nanSafeCompare calls them equal)."""
    nk = len(query.keys)
    kinds = query.field_kinds()
    g, w = sorted(got, key=lambda r: _sort_key(r, nk)), sorted(want, key=lambda r: _sort_key(r, nk))
    assert len(g) == len(w), f"{what}: {len(g)} groups, expected {len(w)}"
    for x, y in zip(g, w):
        assert len(x) == len(y) == len(kinds), f"{what}: row width {len(x)} / {len(y)}"
        for f, (a, b) in enumerate(zip(x, y)):
            if isinstance(a, float) and isinstance(b, float):
                if math.isnan(a) or math.isnan(b):
                    ok = math.isnan(a) and math.isnan(b)
                elif kinds[f] in ("min", "max") and a == 0.0:
                    ok = b == 0.0
                else:
                    ok = _bits(a) == _bits(b)
            else:
                ok = type(a) is type(b) and a == b
            assert ok, f"{what}: group {x[:nk]!r} field {f} ({kinds[f]}): got {a!r}, expected {b!r}"
