"""ctypes mirror of include/snappy_gpu.h plus thin Python handles over it.

The same handle classes drive any library that exports the ABI under a prefix: the product
(`libsnappygpu.so`, prefix ``sd_``) and -- in tests/bench only -- the CPU oracle
(`oracle/liboracle.so`, prefix ``oracle_``), so parity tests feed both the identical descriptors and
ColumnBatch bytes.  Nothing here computes anything: it marshals pointers and sizes.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, List, Optional, Sequence

import numpy as np

from .column_format import ColumnBatch, SqlType, decimal_bytes, parse_row_stream

SD_ABI_VERSION = 2
SD_NUM_METRICS = 12
SD_OPT_RETAIN_BUFFERS = 1
SD_PLAN_MUTATE = 1   # sd_plan_desc.flags: UPDATE / DELETE plan
METRIC_NAMES = ["numOutputRows", "numRowsBuffer", "columnBatchesSeen", "updatedColumnCount",
                "deletedBatchCount", "columnBatchesSkipped", "aggTimeNs", "kernelLaunches",
                "rowsScanned", "algorithmicBytes", "h2dBytes", "scanOutputRows"]
# sdx_plan_launch_log records (include/snappy_gpu.h): SDX_ACC_*, the four batch paths, SDX_REPLAY_*
SDX_LAUNCH_WORDS = 16
LAUNCH_ACCUMULATORS = ["nokey", "private", "shared_atomic", "global_atomic", "hash", "regtable", "rows"]
BATCH_PATHS = ["all_fast", "fast_nulls", "fast_overlay", "general"]
LAUNCH_REPLAYS = [None, "hash_switch", "hash_grow", "rows_grow"]

# sd_status
SD_OK, SD_ERR_INVALID, SD_ERR_UNSUPPORTED, SD_ERR_CUDA, SD_ERR_OVERFLOW, SD_ERR_STATE = range(6)


class SdError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"[sd_status {code}] {msg}")
        self.code = code


# sd_op
class Op:
    COL, LIT = 1, 2
    ADD, SUB, MUL, DIV, NEG, CAST = 10, 11, 12, 13, 14, 15
    EQ, NE, LT, LE, GT, GE = 20, 21, 22, 23, 24, 25
    AND, OR, NOT, ISNULL, ISNOTNULL, IN, STARTSWITH = 30, 31, 32, 33, 34, 35, 36
    PAIR = 37   # (x, y) input of COVAR_POP / COVAR_SAMP / CORR, both DOUBLE; nowhere else
    GROUPING_SET = 38   # INT, a = one grouping-set mask; only in a GROUPING_ID node's list
    GROUPING_ID = 39    # INT, a = first of b GROUPING_SET nodes; only as the last grouping key


class AggFn:
    COUNT_STAR, COUNT, SUM, AVG, MIN, MAX = 1, 2, 3, 4, 5, 6
    # moment aggregates (Spark 2.1.1 CentralMomentAgg) over a DOUBLE input; stddev / variance are the SAMP forms
    STDDEV_POP, STDDEV_SAMP, VAR_POP, VAR_SAMP, SKEWNESS, KURTOSIS = 7, 8, 9, 10, 11, 12
    # two-input aggregates (Spark 2.1.1 Covariance / Corr) over an Op.PAIR node of two DOUBLE inputs
    COVAR_POP, COVAR_SAMP, CORR = 13, 14, 15
    # Spark 2.1.1 First / Last, with ignoreNulls = false / true
    FIRST, LAST, FIRST_IGNORE_NULLS, LAST_IGNORE_NULLS = 16, 17, 18, 19


# partial buffers of a moment aggregate, all non-nullable DOUBLE: [n, avg, m2] + [m3] (SKEWNESS) + [m3, m4] (KURTOSIS)
MOMENT_BUFFERS = {AggFn.STDDEV_POP: 3, AggFn.STDDEV_SAMP: 3, AggFn.VAR_POP: 3, AggFn.VAR_SAMP: 3, AggFn.SKEWNESS: 4, AggFn.KURTOSIS: 5}
# ... and of a two-input aggregate: [n, xAvg, yAvg, ck] + [xMk, yMk] (CORR)
PAIR_BUFFERS = {AggFn.COVAR_POP: 4, AggFn.COVAR_SAMP: 4, AggFn.CORR: 6}
# FIRST / LAST: [value of the input type (nullable), valueSet BOOLEAN]
ORDER_AGGS = (AggFn.FIRST, AggFn.LAST, AggFn.FIRST_IGNORE_NULLS, AggFn.LAST_IGNORE_NULLS)


class sd_column(C.Structure):
    _fields_ = [("type", C.c_int32), ("nullable", C.c_int32), ("table_ordinal", C.c_int32), ("scale", C.c_int32),
                ("precision", C.c_int32)]


class sd_expr(C.Structure):
    _fields_ = [("op", C.c_int32), ("type", C.c_int32), ("a", C.c_int32), ("b", C.c_int32), ("c", C.c_int32)]


class sd_agg(C.Structure):
    _fields_ = [("fn", C.c_int32), ("expr", C.c_int32)]


class sd_plan_desc(C.Structure):
    _fields_ = [("abi_version", C.c_int32),
                ("ncols", C.c_int32), ("cols", C.POINTER(sd_column)),
                ("nexprs", C.c_int32), ("exprs", C.POINTER(sd_expr)),
                ("filter", C.c_int32),
                ("nkeys", C.c_int32), ("keys", C.POINTER(C.c_int32)),
                ("naggs", C.c_int32), ("aggs", C.POINTER(sd_agg)),
                ("nproj", C.c_int32), ("proj", C.POINTER(C.c_int32)),
                ("nliterals", C.c_int32), ("literal_types", C.POINTER(C.c_int32)),
                ("flags", C.c_int32)]


class sd_literal(C.Structure):
    _fields_ = [("type", C.c_int32), ("is_null", C.c_int32), ("i", C.c_int64), ("d", C.c_double),
                ("s", C.c_char_p), ("slen", C.c_int32), ("pad_", C.c_int32)]


class sd_raw_column(C.Structure):
    _fields_ = [("values", C.c_void_p), ("str_bytes", C.c_void_p), ("nulls", C.c_void_p)]


class sd_batch(C.Structure):
    _fields_ = [("num_rows", C.c_int32), ("ncols", C.c_int32),
                ("col_bufs", C.POINTER(C.c_void_p)), ("col_lens", C.POINTER(C.c_int64)),
                ("delta0", C.POINTER(C.c_void_p)), ("delta0_lens", C.POINTER(C.c_int64)),
                ("delta1", C.POINTER(C.c_void_p)), ("delta1_lens", C.POINTER(C.c_int64)),
                ("delete_buf", C.c_void_p), ("delete_len", C.c_int64),
                ("stats_row", C.c_void_p), ("stats_len", C.c_int64),
                ("stats_ncols", C.c_int32), ("bucket_id", C.c_int32), ("batch_id", C.c_int64)]


def _buf_ptr(b) -> int:
    """Address of a bytes / bytearray / numpy buffer without copying."""
    if b is None:
        return 0
    if isinstance(b, np.ndarray):
        return b.ctypes.data
    if isinstance(b, bytes):
        return C.cast(C.c_char_p(b), C.c_void_p).value or 0
    if isinstance(b, (bytearray, memoryview)):
        return C.addressof((C.c_char * len(b)).from_buffer(b))
    if isinstance(b, int):
        return b
    raise TypeError(type(b))


def _buf_len(b) -> int:
    if b is None:
        return 0
    if isinstance(b, np.ndarray):
        return b.nbytes
    return len(b)


class MarshalledBatch:
    """An sd_batch plus the Python objects that keep its pointers alive.
    ``cols`` selects table columns (plan scan order); ``None`` keeps the table's own order/width
    (what sd_store_put_batch wants)."""

    def __init__(self, batch: ColumnBatch, cols: Optional[Sequence[int]] = None, stats_ncols: Optional[int] = None):
        idx = list(range(len(batch.columns))) if cols is None else list(cols)
        n = len(idx)
        self._keep = [batch]
        self.col_bufs = (C.c_void_p * n)(*[_buf_ptr(batch.columns[c]) for c in idx])
        self.col_lens = (C.c_int64 * n)(*[_buf_len(batch.columns[c]) for c in idx])
        self.d0 = (C.c_void_p * n)(*[_buf_ptr(batch.delta0.get(c)) for c in idx])
        self.d0l = (C.c_int64 * n)(*[_buf_len(batch.delta0.get(c)) for c in idx])
        self.d1 = (C.c_void_p * n)(*[_buf_ptr(batch.delta1.get(c)) for c in idx])
        self.d1l = (C.c_int64 * n)(*[_buf_len(batch.delta1.get(c)) for c in idx])
        b = sd_batch()
        b.num_rows = batch.num_rows
        b.ncols = n
        b.col_bufs = C.cast(self.col_bufs, C.POINTER(C.c_void_p))
        b.col_lens = C.cast(self.col_lens, C.POINTER(C.c_int64))
        b.delta0 = C.cast(self.d0, C.POINTER(C.c_void_p))
        b.delta0_lens = C.cast(self.d0l, C.POINTER(C.c_int64))
        b.delta1 = C.cast(self.d1, C.POINTER(C.c_void_p))
        b.delta1_lens = C.cast(self.d1l, C.POINTER(C.c_int64))
        b.delete_buf = _buf_ptr(batch.delete_mask)
        b.delete_len = _buf_len(batch.delete_mask)
        b.stats_row = _buf_ptr(batch.stats)
        b.stats_len = _buf_len(batch.stats)
        b.stats_ncols = stats_ncols if stats_ncols is not None else len(batch.columns)
        b.bucket_id = batch.bucket_id
        b.batch_id = batch.batch_id
        self.c = b


def make_literal(t: SqlType, v, wide: bool = False) -> sd_literal:
    """`wide`: the slot holds a DECIMAL of more than 18 digits; an int value is passed as its BigInteger bytes."""
    lit = sd_literal()
    lit.type = int(t)
    if v is None:
        lit.is_null = 1
        return lit
    t = SqlType(t)
    if wide:
        b = bytes(v) if isinstance(v, (bytes, bytearray)) else decimal_bytes(int(v))
        lit.s = b
        lit.slen = len(b)
    elif t == SqlType.STRING:
        b = v if isinstance(v, bytes) else str(v).encode("utf-8")
        lit.s = b
        lit.slen = len(b)
    elif t in (SqlType.FLOAT, SqlType.DOUBLE):
        lit.d = float(v)
    else:
        lit.i = int(v)
    return lit


class Api:
    """Function table of one library exporting the ABI under ``prefix``."""

    def __init__(self, path: str, prefix: str):
        self.lib = C.CDLL(path, mode=C.RTLD_GLOBAL if prefix == "sd_" else C.RTLD_LOCAL)
        self.prefix = prefix
        self.path = path
        L = self.lib
        vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64

        def fn(name, restype, *argtypes, required=True):
            try:
                f = getattr(L, prefix + name)
            except AttributeError:
                if required:
                    raise
                return None
            f.restype = restype
            f.argtypes = list(argtypes)
            return f

        self.last_error = fn("last_error", C.c_char_p)
        self.plan_create = fn("plan_create", C.c_int, C.POINTER(sd_plan_desc), C.POINTER(vp))
        self.plan_set_literals = fn("plan_set_literals", C.c_int, vp, C.POINTER(sd_literal), i32)
        self.batch_submit = fn("batch_submit", C.c_int, vp, C.POINTER(sd_batch))
        self.rows_submit = fn("rows_submit", C.c_int, vp, vp, i64, i32)
        self.plan_finish = fn("plan_finish", C.c_int, vp, vp, i64, C.POINTER(i64), C.POINTER(i64))
        self.plan_reset = fn("plan_reset", C.c_int, vp)
        self.plan_metrics = fn("plan_metrics", C.c_int, vp, C.POINTER(i64))
        self.plan_destroy = fn("plan_destroy", None, vp)
        self.final_merge = fn("final_merge", C.c_int, C.POINTER(sd_plan_desc), vp, i64, vp, i64,
                              C.POINTER(i64), C.POINTER(i64))
        # product-only entry points
        self.init = fn("init", C.c_int, C.c_int, required=False)
        self.device_count = fn("device_count", C.c_int, C.POINTER(C.c_int), required=False)
        self.version = fn("version", C.c_char_p, required=False)
        self.plan_set_stream = fn("plan_set_stream", C.c_int, vp, vp, required=False)
        self.plan_set_option = fn("plan_set_option", C.c_int, vp, i32, i64, required=False)
        self.plan_kernel_name = fn("plan_kernel_name", C.c_char_p, vp, required=False)
        self.store_create = fn("store_create", C.c_int, C.c_int, i32, C.POINTER(sd_column), C.POINTER(vp), required=False)
        self.store_put_batch = fn("store_put_batch", C.c_int, vp, C.POINTER(sd_batch), required=False)
        self.store_encode_batch = fn("store_encode_batch", C.c_int, vp, i32, C.POINTER(sd_raw_column), i32, i32, i64, required=False)
        self.store_num_batches = fn("store_num_batches", C.c_int, vp, C.POINTER(i64), required=False)
        self.store_bytes = fn("store_bytes", C.c_int, vp, C.POINTER(i64), required=False)
        self.plan_scan_store = fn("plan_scan_store", C.c_int, vp, vp, C.POINTER(i32), i32, required=False)
        self.store_destroy = fn("store_destroy", None, vp, required=False)
        self.plan_final_merge = fn("plan_final_merge", C.c_int, vp, vp, i64, vp, i64, C.POINTER(i64), C.POINTER(i64), required=False)
        self.plan_partials_layout = fn("plan_partials_layout", C.c_int, vp, C.POINTER(i32), C.POINTER(i32),
                                       C.POINTER(i32), required=False)
        self.partial_merge = fn("partial_merge", C.c_int, C.POINTER(sd_plan_desc), vp, i64, vp, i64, C.POINTER(i64), C.POINTER(i64), required=False)
        self.plan_partial_merge = fn("plan_partial_merge", C.c_int, vp, vp, i64, vp, i64, C.POINTER(i64), C.POINTER(i64), required=False)
        self.comm_unique_id = fn("comm_unique_id", C.c_int, vp, required=False)
        self.comm_create = fn("comm_create", C.c_int, vp, i32, i32, i32, C.POINTER(vp), required=False)
        self.comm_destroy = fn("comm_destroy", None, vp, required=False)
        self.comm_info = fn("comm_info", C.c_int, vp, C.POINTER(i64), required=False)
        self.plan_exchange = fn("plan_exchange", C.c_int, vp, vp, required=False)
        self.plan_execute_store = fn("plan_execute_store", C.c_int, vp, vp, C.POINTER(i32), i32, C.POINTER(sd_literal), i32, vp,
                                     vp, i64, C.POINTER(i64), C.POINTER(i64), required=False)
        self.host_alloc = fn("host_alloc", C.c_int, i64, C.POINTER(vp), required=False)
        self.host_free = fn("host_free", None, vp, required=False)
        self.plan_export_partials = fn("plan_export_partials", C.c_int, vp, vp, i64, required=False)
        self.plan_import_partials = fn("plan_import_partials", C.c_int, vp, vp, i64, required=False)
        self.plan_update_store = fn("plan_update_store", C.c_int, vp, vp, C.POINTER(i32), i32, C.POINTER(sd_literal), i32,
                                    C.POINTER(i32), C.POINTER(i64), required=False)
        self.plan_delete_store = fn("plan_delete_store", C.c_int, vp, vp, C.POINTER(i32), i32, C.POINTER(sd_literal), i32,
                                    C.POINTER(i64), required=False)

    def check(self, rc: int):
        if rc != 0:
            msg = self.last_error()
            raise SdError(rc, msg.decode("utf-8", "replace") if msg else "unknown error")


_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG_DIR, "csrc", "libsnappygpu.so")
_product: Optional[Api] = None


def product_api() -> Api:
    """The CUDA library.  Fails loudly when it has not been built: there is no CPU fallback."""
    global _product
    if _product is None:
        if not os.path.exists(LIB_PATH):
            raise SdError(SD_ERR_STATE, f"{LIB_PATH} not built -- run `python -c 'import __graft_entry__ as g; g.build()'`; "
                                        "there is no CPU fallback")
        _product = Api(LIB_PATH, "sd_")
        # extension entry points (sdx_*)
        L = _product.lib
        L.sdx_store_gen_lineitem.restype = C.c_int
        L.sdx_store_gen_lineitem.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_uint64, C.c_int32]
        L.sdx_store_get_buffer.restype = C.c_int
        L.sdx_store_get_buffer.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]
        L.sdx_store_batch_info.restype = C.c_int
        L.sdx_store_batch_info.argtypes = [C.c_void_p, C.c_int64, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int64)]
        L.sdx_store_memory_info.restype = C.c_int
        L.sdx_store_memory_info.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.sdx_store_image_info.restype = C.c_int
        L.sdx_store_image_info.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
        L.sdx_image_width.restype = C.c_int
        L.sdx_image_width.argtypes = [C.c_int32, C.c_int32, C.c_uint64, C.c_int64, C.c_int64, C.POINTER(C.c_int32)]
        L.sdx_store_get_delta.restype = C.c_int
        L.sdx_store_get_delta.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]
        L.sdx_store_get_deletes.restype = C.c_int
        L.sdx_store_get_deletes.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]
        L.sdx_plan_rollup_info.restype = C.c_int
        L.sdx_plan_rollup_info.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
        L.sdx_last_mutation_timing.restype = C.c_int
        L.sdx_last_mutation_timing.argtypes = [C.POINTER(C.c_double)]
        L.sd_store_compact.restype = C.c_int
        L.sd_store_compact.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.c_int32, C.c_double, C.POINTER(C.c_int64)]
        L.sdx_last_compaction_timing.restype = C.c_int
        L.sdx_last_compaction_timing.argtypes = [C.POINTER(C.c_double)]
        L.sd_store_reclaim.restype = C.c_int
        L.sd_store_reclaim.argtypes = [C.c_void_p, C.c_double, C.POINTER(C.c_int64)]
        L.sdx_last_reclaim_timing.restype = C.c_int
        L.sdx_last_reclaim_timing.argtypes = [C.POINTER(C.c_double)]
        L.sdx_store_extent_bytes.restype = C.c_int
        L.sdx_store_extent_bytes.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
        L.sdx_plan_launch_log.restype = C.c_int
        L.sdx_plan_launch_log.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.c_int32, C.POINTER(C.c_int32)]
    return _product


class PlanDesc:
    """Owns the ctypes arrays behind an sd_plan_desc."""

    def __init__(self, cols, exprs, filter_node, keys, aggs, proj, literal_types, flags: int = 0, targets: Sequence[int] = ()):
        self.flags = int(flags)              # SD_PLAN_MUTATE: UPDATE / DELETE
        self.targets = list(targets)         # UPDATE: table ordinal that proj[i] writes
        self.cols_py = list(cols)            # (SqlType, nullable, table_ordinal[, scale])
        self.exprs_py = list(exprs)          # (op, type, a, b, c)
        self.keys_py = list(keys)
        self.aggs_py = list(aggs)            # (fn, expr)
        self.proj_py = list(proj)
        self.literal_types_py = [SqlType(t) for t in literal_types]
        self.filter = filter_node
        # literal slots of a DECIMAL wider than 18 digits: a LIT node of that type, or an IN list over such an operand
        self.lit_wide = [False] * len(self.literal_types_py)
        for i, (op, t, a, b, c) in enumerate(self.exprs_py):
            if op == Op.LIT and self._wide(i):
                self.lit_wide[a] = True
            if op == Op.IN and self._wide(a):
                for k in range(c):
                    self.lit_wide[b + k] = True
        self._cols = (sd_column * max(1, len(self.cols_py)))()
        for i, c in enumerate(self.cols_py):
            self._cols[i] = sd_column(int(c[0]), int(bool(c[1])), int(c[2]), int(c[3]) if len(c) > 3 else 0,
                                      int(c[4]) if len(c) > 4 else (18 if int(c[0]) == int(SqlType.DECIMAL) else 0))
        self._exprs = (sd_expr * max(1, len(self.exprs_py)))()
        for i, e in enumerate(self.exprs_py):
            self._exprs[i] = sd_expr(*[int(x) for x in e])
        self._keys = (C.c_int32 * max(1, len(self.keys_py)))(*self.keys_py)
        self._aggs = (sd_agg * max(1, len(self.aggs_py)))()
        for i, a in enumerate(self.aggs_py):
            self._aggs[i] = sd_agg(int(a[0]), int(a[1]))
        self._proj = (C.c_int32 * max(1, len(self.proj_py)))(*self.proj_py)
        self._lt = (C.c_int32 * max(1, len(self.literal_types_py)))(*[int(t) for t in self.literal_types_py])
        d = sd_plan_desc()
        d.abi_version = SD_ABI_VERSION
        d.ncols, d.cols = len(self.cols_py), C.cast(self._cols, C.POINTER(sd_column))
        d.nexprs, d.exprs = len(self.exprs_py), C.cast(self._exprs, C.POINTER(sd_expr))
        d.filter = filter_node
        d.nkeys, d.keys = len(self.keys_py), C.cast(self._keys, C.POINTER(C.c_int32))
        d.naggs, d.aggs = len(self.aggs_py), C.cast(self._aggs, C.POINTER(sd_agg))
        d.nproj, d.proj = len(self.proj_py), C.cast(self._proj, C.POINTER(C.c_int32))
        d.nliterals, d.literal_types = len(self.literal_types_py), C.cast(self._lt, C.POINTER(C.c_int32))
        d.flags = self.flags
        self.c = d

    @property
    def table_cols(self) -> List[int]:
        return [c[2] for c in self.cols_py]

    # -- schemas of the rows the plan emits ----------------------------------------------------
    # a field is a SqlType, or (SqlType.DECIMAL, precision, scale): Spark 2.1.1 Sum / Average over DECIMAL(p,s) have the
    # buffer DECIMAL(p+10,s); Average's result is DECIMAL(p+4,s+4)
    def _ps(self, node: int):
        op, _, a, _, c = self.exprs_py[node]
        if op == Op.COL:
            col = self.cols_py[a]
            return (col[4] if len(col) > 4 else 18), (col[3] if len(col) > 3 else 0)
        if op == Op.NEG:
            return self._ps(a)
        return c >> 8, c & 0xFF

    def _wide(self, node: int) -> bool:
        return SqlType(self.exprs_py[node][1]) == SqlType.DECIMAL and self._ps(node)[0] > 18

    def _ftype(self, node: int):
        t = SqlType(self.exprs_py[node][1])
        return (t,) + self._ps(node) if t == SqlType.DECIMAL else t

    def _sum_type(self, node: int):
        t = SqlType(self.exprs_py[node][1])
        if t == SqlType.DECIMAL:
            p, s = self._ps(node)
            return (SqlType.DECIMAL, min(38, p + 10), s)
        return SqlType.DOUBLE if t in (SqlType.FLOAT, SqlType.DOUBLE) else SqlType.LONG

    def partial_schema(self) -> List[object]:
        if not self.aggs_py and not self.keys_py:
            return [self._ftype(n) for n in self.proj_py]
        out = [self._ftype(k) for k in self.keys_py]
        for fn, e in self.aggs_py:
            if fn in (AggFn.COUNT_STAR, AggFn.COUNT):
                out.append(SqlType.LONG)
            elif fn == AggFn.SUM:
                out.append(self._sum_type(e))
            elif fn == AggFn.AVG:
                st = self._sum_type(e)
                out += [st if isinstance(st, tuple) else SqlType.DOUBLE, SqlType.LONG]
            elif fn in MOMENT_BUFFERS:
                out += [SqlType.DOUBLE] * MOMENT_BUFFERS[fn]
            elif fn in PAIR_BUFFERS:
                out += [SqlType.DOUBLE] * PAIR_BUFFERS[fn]
            elif fn in ORDER_AGGS:
                out += [self._ftype(e), SqlType.BOOLEAN]
            else:
                out.append(self._ftype(e))
        return out

    def final_schema(self) -> List[object]:
        out = [self._ftype(k) for k in self.keys_py]
        for fn, e in self.aggs_py:
            if fn in (AggFn.COUNT_STAR, AggFn.COUNT):
                out.append(SqlType.LONG)
            elif fn == AggFn.SUM:
                out.append(self._sum_type(e))
            elif fn == AggFn.AVG:
                if SqlType(self.exprs_py[e][1]) == SqlType.DECIMAL:
                    p, s = self._ps(e)
                    out.append((SqlType.DECIMAL, min(38, p + 4), min(38, s + 4)))
                else:
                    out.append(SqlType.DOUBLE)
            elif fn in MOMENT_BUFFERS or fn in PAIR_BUFFERS:
                out.append(SqlType.DOUBLE)
            else:
                out.append(self._ftype(e))
        return out


class Plan:
    """One execution handle (one Spark task / partition)."""

    def __init__(self, api: Api, desc: PlanDesc):
        self.api, self.desc = api, desc
        h = C.c_void_p()
        api.check(api.plan_create(C.byref(desc.c), C.byref(h)))
        self.h = h
        self._lits = None

    def literal_array(self, values: Sequence[object]):
        n = len(values)
        arr = (sd_literal * max(1, n))()
        for i, v in enumerate(values):
            arr[i] = make_literal(self.desc.literal_types_py[i], v, self.desc.lit_wide[i])
        return arr

    def set_literals(self, values: Sequence[object]):
        arr = self.literal_array(values)
        self._lits = arr
        self.api.check(self.api.plan_set_literals(self.h, arr, len(values)))
        return self

    def execute_store_raw(self, store: "Store", lit_array, nlits: int, comm: Optional["Comm"] = None) -> bytes:
        """One execution of the cached plan over a resident store in ONE C call (sd_plan_execute_store): reset, literals,
        scan, the NCCL exchange when `comm` is given, partial rows (merged over the ranks with `comm`)."""
        if getattr(self, "_out_buf", None) is None:
            self._out_buf = C.create_string_buffer(1 << 14)
        if getattr(self, "_out_len", None) is None:
            self._out_len, self._out_rows = C.c_int64(), C.c_int64()
        rc = self.api.plan_execute_store(self.h, store.h, None, 0, lit_array, nlits, comm.h if comm is not None else None,
                                         self._out_buf, len(self._out_buf), C.byref(self._out_len), C.byref(self._out_rows))
        if rc == SD_ERR_OVERFLOW:   # the execution is complete; only the caller's buffer was too small
            self._out_buf = C.create_string_buffer(int(self._out_len.value) + 64)
            return self.finish_raw()
        if rc:
            self.api.check(rc)
        return C.string_at(self._out_buf, self._out_len.value)

    def _pinned_out(self, need: int):
        """Page-locked result buffer owned by this handle (sd_host_alloc): the projected rows of MODE_PROJECT arrive in it by one
        device->host copy at link speed."""
        if getattr(self, "_pin_cap", 0) < need:
            if getattr(self, "_pin_ptr", None):
                self.api.host_free(self._pin_ptr)
                self._pin_ptr, self._pin_cap = None, 0
            ptr = C.c_void_p()
            cap = int(need) + int(need) // 4 + (1 << 16)
            self.api.check(self.api.host_alloc(cap, C.byref(ptr)))
            self._pin_ptr, self._pin_cap = ptr, cap
        return self._pin_ptr, self._pin_cap

    def execute_store_view(self, store: "Store", lit_array, nlits: int, comm: Optional["Comm"] = None) -> memoryview:
        """execute_store_raw without the two host copies: the row stream lands in this handle's page-locked buffer and comes
        back as a memoryview of it (valid until the next execution on this handle)."""
        if getattr(self, "_out_len", None) is None:
            self._out_len, self._out_rows = C.c_int64(), C.c_int64()
        ptr, cap = self._pinned_out(1 << 20)
        rc = self.api.plan_execute_store(self.h, store.h, None, 0, lit_array, nlits, comm.h if comm is not None else None,
                                         ptr, cap, C.byref(self._out_len), C.byref(self._out_rows))
        if rc == SD_ERR_OVERFLOW:   # the execution is complete; only the buffer was too small
            ptr, cap = self._pinned_out(int(self._out_len.value) + 64)
            rc = self.api.plan_finish(self.h, ptr, cap, C.byref(self._out_len), C.byref(self._out_rows))
        if rc:
            self.api.check(rc)
        n = int(self._out_len.value)
        return memoryview((C.c_char * max(n, 1)).from_address(ptr.value)).cast("B")[:n]

    def exchange(self, comm: "Comm"):
        self.api.check(self.api.plan_exchange(self.h, comm.h))
        return self

    def partial_merge_raw(self, partial_raw: bytes) -> bytes:
        cap = max(1 << 14, 2 * len(partial_raw) + 1024)
        buf = C.create_string_buffer(cap)
        out_len, out_rows = C.c_int64(), C.c_int64()
        self.api.check(self.api.plan_partial_merge(self.h, _buf_ptr(partial_raw), len(partial_raw), buf, cap, C.byref(out_len), C.byref(out_rows)))
        return buf.raw[: out_len.value]

    def submit(self, batch: ColumnBatch):
        mb = MarshalledBatch(batch, self.desc.table_cols)
        self.api.check(self.api.batch_submit(self.h, C.byref(mb.c)))
        return self

    def submit_marshalled(self, mb: MarshalledBatch):
        self.api.check(self.api.batch_submit(self.h, C.byref(mb.c)))
        return self

    def submit_rows(self, rows: bytes, nrows: int):
        self.api.check(self.api.rows_submit(self.h, _buf_ptr(rows), len(rows), nrows))
        return self

    def scan_store(self, store: "Store", buckets: Optional[Sequence[int]] = None):
        if buckets is None:
            self.api.check(self.api.plan_scan_store(self.h, store.h, None, 0))
        else:
            arr = (C.c_int32 * len(buckets))(*buckets)
            self.api.check(self.api.plan_scan_store(self.h, store.h, arr, len(buckets)))
        return self

    def _mutation_args(self, store: "Store", lits: Sequence[object], buckets: Optional[Sequence[int]]):
        arr = self.literal_array(lits)
        b = (C.c_int32 * max(1, len(buckets or ())))(*(buckets or ()))
        return arr, b, len(buckets or ())

    def update_store(self, store: "Store", lits: Sequence[object] = (), buckets: Optional[Sequence[int]] = None) -> int:
        """UPDATE store SET targets = proj WHERE filter, on the device (sd_plan_update_store) -> rows updated."""
        arr, b, nb = self._mutation_args(store, lits, buckets)
        tg = (C.c_int32 * max(1, len(self.desc.targets)))(*self.desc.targets)
        rows = C.c_int64()
        self.api.check(self.api.plan_update_store(self.h, store.h, b if nb else None, nb, arr, len(lits), tg, C.byref(rows)))
        return int(rows.value)

    def delete_store(self, store: "Store", lits: Sequence[object] = (), buckets: Optional[Sequence[int]] = None) -> int:
        """DELETE FROM store WHERE filter, on the device (sd_plan_delete_store) -> rows deleted."""
        arr, b, nb = self._mutation_args(store, lits, buckets)
        rows = C.c_int64()
        self.api.check(self.api.plan_delete_store(self.h, store.h, b if nb else None, nb, arr, len(lits), C.byref(rows)))
        return int(rows.value)

    def finish_raw(self) -> bytes:
        while True:
            if getattr(self, "_out_buf", None) is None:
                self._out_buf = C.create_string_buffer(1 << 14)
            buf = self._out_buf
            out_len, out_rows = C.c_int64(), C.c_int64()
            rc = self.api.plan_finish(self.h, buf, len(buf), C.byref(out_len), C.byref(out_rows))
            if rc == SD_ERR_OVERFLOW:
                self._out_buf = C.create_string_buffer(int(out_len.value) + 64)
                continue
            self.api.check(rc)
            return buf.raw[: out_len.value]

    def finish(self) -> List[List[object]]:
        return parse_row_stream(self.finish_raw(), self.desc.partial_schema())

    def reset(self):
        self.api.check(self.api.plan_reset(self.h))
        return self

    def final_merge_raw(self, partial_raw: bytes) -> bytes:
        """Final merge of partial rows (all partitions) reusing this handle's plan analysis -> final row stream."""
        cap = max(1 << 14, 4 * len(partial_raw) + 1024)
        if getattr(self, "_merge_buf", None) is None or len(self._merge_buf) < cap:
            self._merge_buf = C.create_string_buffer(cap)
        out_len, out_rows = C.c_int64(), C.c_int64()
        self.api.check(self.api.plan_final_merge(self.h, _buf_ptr(partial_raw), len(partial_raw), self._merge_buf, cap,
                                                 C.byref(out_len), C.byref(out_rows)))
        return self._merge_buf.raw[: out_len.value]

    def final_merge(self, partial_raw: bytes) -> List[List[object]]:
        return parse_row_stream(self.final_merge_raw(partial_raw), self.desc.final_schema())

    def metrics(self) -> Dict[str, int]:
        out = (C.c_int64 * SD_NUM_METRICS)()
        self.api.check(self.api.plan_metrics(self.h, out))
        return dict(zip(METRIC_NAMES, list(out)))

    def kernel_name(self) -> str:
        return self.api.plan_kernel_name(self.h).decode()

    def launch_log(self) -> List[Dict[str, object]]:
        """What every kernel launch since the last reset ran (sdx_plan_launch_log), one dict per launch in launch order."""
        f = self.api.lib.sdx_plan_launch_log
        n = C.c_int32()
        rc = f(self.h, None, 0, C.byref(n))
        if rc not in (SD_OK, SD_ERR_OVERFLOW):
            self.api.check(rc)
        buf = (C.c_int64 * max(1, n.value * SDX_LAUNCH_WORDS))()
        self.api.check(f(self.h, buf, n.value, C.byref(n)))
        out = []
        for i in range(n.value):
            w = buf[i * SDX_LAUNCH_WORDS:(i + 1) * SDX_LAUNCH_WORDS]
            out.append({"accumulator": LAUNCH_ACCUMULATORS[w[0]], "full_paths": bool(w[1]), "literal_nulls": bool(w[2]),
                        "nstages": w[3], "tile_rows": w[4], "chunk_rows": w[5], "grid": w[6], "ngroups": w[7],
                        "paths": dict(zip(BATCH_PATHS, w[8:12])), "replay": LAUNCH_REPLAYS[w[12]],
                        "nbatches": w[13], "chunks": w[14], "streamed_bytes": w[15]})
        return out

    def rollup_info(self) -> Dict[str, float]:
        """The grouping-sets roll-up of the last execution (sdx_plan_rollup_info)."""
        out = (C.c_double * 4)()
        self.api.check(self.api.lib.sdx_plan_rollup_info(self.h, out))
        return {"ms": out[0], "fine": int(out[1]), "coarse": int(out[2]), "launches": int(out[3])}

    def set_option(self, option: int, value: int):
        self.api.check(self.api.plan_set_option(self.h, option, value))
        return self

    def set_stream(self, stream_ptr: int):
        self.api.check(self.api.plan_set_stream(self.h, stream_ptr))

    def close(self):
        if self.h:
            self.api.plan_destroy(self.h)
            self.h = None
        if getattr(self, "_pin_ptr", None):
            self.api.host_free(self._pin_ptr)
            self._pin_ptr, self._pin_cap = None, 0

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def final_merge(api: Api, desc: PlanDesc, partial_raw: bytes) -> List[List[object]]:
    cap = max(1 << 16, 4 * len(partial_raw) + 1024)
    buf = C.create_string_buffer(cap)
    out_len, out_rows = C.c_int64(), C.c_int64()
    api.check(api.final_merge(C.byref(desc.c), _buf_ptr(partial_raw), len(partial_raw), buf, cap,
                              C.byref(out_len), C.byref(out_rows)))
    return parse_row_stream(buf.raw[: out_len.value], desc.final_schema())


def partial_merge_raw(api: Api, desc: PlanDesc, partial_raw: bytes) -> bytes:
    """Merged PARTIAL rows (host only: sd_partial_merge)."""
    cap = max(1 << 16, 2 * len(partial_raw) + 1024)
    buf = C.create_string_buffer(cap)
    out_len, out_rows = C.c_int64(), C.c_int64()
    api.check(api.partial_merge(C.byref(desc.c), _buf_ptr(partial_raw), len(partial_raw), buf, cap, C.byref(out_len), C.byref(out_rows)))
    return buf.raw[: out_len.value]


class Comm:
    """sd_comm: the NCCL communicator of the partial -> final exchange.  `broadcast_bytes(b: bytes | None) -> bytes` moves
    rank 0's 128-byte id to every rank (torch.distributed.broadcast_object_list, a Spark broadcast, ...)."""

    def __init__(self, api: Api, rank: int, world: int, device: int, broadcast_bytes):
        self.api = api
        ident = None
        if rank == 0:
            buf = C.create_string_buffer(128)
            api.check(api.comm_unique_id(buf))
            ident = buf.raw
        ident = broadcast_bytes(ident)
        assert len(ident) == 128
        h = C.c_void_p()
        api.check(api.comm_create(ident, rank, world, device, C.byref(h)))
        self.h = h

    def info(self):
        out = (C.c_int64 * 4)()
        self.api.check(self.api.comm_info(self.h, out))
        return {"world": out[0], "slot_bytes": out[1], "all_gathers": out[2], "regrows": out[3]}

    def close(self):
        if self.h:
            self.api.comm_destroy(self.h)
            self.h = None


class Store:
    """Device-resident column store handle (product only)."""

    def __init__(self, api: Api, schema, device: int = 0):
        """schema: [(SqlType, nullable[, precision, scale])] per table column, in table order (DECIMAL precision
        defaults to 18)."""
        self.api = api
        self.schema = [(SqlType(c[0]), bool(c[1])) for c in schema]
        arr = (sd_column * max(1, len(self.schema)))()
        for i, c in enumerate(schema):
            t, n = int(c[0]), int(bool(c[1]))
            prec, scale = (int(c[2]), int(c[3])) if len(c) > 3 else (18 if t == int(SqlType.DECIMAL) else 0, 0)
            arr[i] = sd_column(t, n, i, scale, prec)
        h = C.c_void_p()
        api.check(api.store_create(device, len(self.schema), arr, C.byref(h)))
        self.h = h

    def put(self, batch: ColumnBatch):
        mb = MarshalledBatch(batch, None)
        self.api.check(self.api.store_put_batch(self.h, C.byref(mb.c)))

    def encode_batch(self, num_rows: int, raw: Dict[int, tuple], bucket_id: int = 0, batch_id: int = 0):
        """Ingest: raw column values -> encoded ColumnBatch ON THE DEVICE (sd_store_encode_batch).
        raw[table_col] = (values, nulls) with values a numpy array of the column's type (STRING: a sequence of bytes),
        nulls a bool array or None."""
        arr = (sd_raw_column * max(1, len(self.schema)))()
        keep = []
        for c, (vals, nulls) in raw.items():
            t = self.schema[c][0]
            if t == SqlType.STRING:
                bs = [bytes(v) if v is not None else b"" for v in vals]
                offs = np.zeros(len(bs) + 1, dtype=np.int32)
                np.cumsum([len(b) for b in bs], out=offs[1:])
                blob = np.frombuffer(b"".join(bs) + b"\0", dtype=np.uint8)
                keep += [offs, blob]
                arr[c].values, arr[c].str_bytes = offs.ctypes.data, blob.ctypes.data
            else:
                from .column_format import np_dtype
                v = np.ascontiguousarray(np.asarray(vals).astype(bool).astype("u1") if t == SqlType.BOOLEAN else np.asarray(vals).astype(np_dtype(t)))
                keep.append(v)
                arr[c].values = v.ctypes.data
            if nulls is not None:
                nb = np.ascontiguousarray(np.asarray(nulls).astype("u1"))
                keep.append(nb)
                arr[c].nulls = nb.ctypes.data
        self.api.check(self.api.store_encode_batch(self.h, num_rows, arr, len(self.schema), bucket_id, batch_id))

    def get_stats(self, batch_index: int) -> bytes:
        f = self.api.lib.sdx_store_get_stats
        f.restype = C.c_int
        f.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]
        ln = C.c_int64()
        buf = C.create_string_buffer(1 << 16)
        self.api.check(f(self.h, batch_index, buf, len(buf), C.byref(ln)))
        return buf.raw[: ln.value]

    def num_batches(self) -> int:
        out = C.c_int64()
        self.api.check(self.api.store_num_batches(self.h, C.byref(out)))
        return out.value

    def nbytes(self) -> int:
        out = C.c_int64()
        self.api.check(self.api.store_bytes(self.h, C.byref(out)))
        return out.value

    def gen_lineitem(self, first_row: int, nrows: int, rows_per_batch: int, nbuckets: int, seed: int, column_mask: int):
        self.api.check(self.api.lib.sdx_store_gen_lineitem(self.h, first_row, nrows, rows_per_batch, nbuckets, seed, column_mask))

    def get_buffer(self, batch_index: int, table_col: int) -> bytes:
        ln = C.c_int64()
        rc = self.api.lib.sdx_store_get_buffer(self.h, batch_index, table_col, None, 0, C.byref(ln))
        if rc not in (0, SD_ERR_OVERFLOW):
            self.api.check(rc)
        buf = C.create_string_buffer(max(1, ln.value))
        self.api.check(self.api.lib.sdx_store_get_buffer(self.h, batch_index, table_col, buf, ln.value, C.byref(ln)))
        return buf.raw[: ln.value]

    def batch_info(self, batch_index: int):
        n, b, i = C.c_int32(), C.c_int32(), C.c_int64()
        self.api.check(self.api.lib.sdx_store_batch_info(self.h, batch_index, C.byref(n), C.byref(b), C.byref(i)))
        return n.value, b.value, i.value

    def memory_info(self):
        """(compressible bytes, slab bytes) of the device memory the store holds."""
        comp, total = C.c_int64(), C.c_int64()
        self.api.check(self.api.lib.sdx_store_memory_info(self.h, C.byref(comp), C.byref(total)))
        return comp.value, total.value

    def image_info(self) -> Dict[str, int]:
        """Scan images of the current batch versions (sdx_store_image_info)."""
        out = (C.c_int64 * 4)()
        self.api.check(self.api.lib.sdx_store_image_info(self.h, out))
        return {"bytes": out[0], "images": out[1], "mismatches": out[2], "build_us": out[3]}

    def close(self):
        if self.h:
            self.api.store_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def get_delta(self, batch_index: int, table_col: int, depth: int = 0) -> bytes:
        """A resident update delta in the reference's byte layout (sdx_store_get_delta)."""
        ln = C.c_int64()
        rc = self.api.lib.sdx_store_get_delta(self.h, batch_index, table_col, depth, None, 0, C.byref(ln))
        if rc not in (0, SD_ERR_OVERFLOW):
            self.api.check(rc)
        buf = C.create_string_buffer(max(1, ln.value))
        self.api.check(self.api.lib.sdx_store_get_delta(self.h, batch_index, table_col, depth, buf, len(buf), C.byref(ln)))
        return buf.raw[: ln.value]

    def compact(self, min_dirty_fraction: float = 0.0, buckets: Optional[Sequence[int]] = None) -> Dict[str, int]:
        """Fold the update deltas and delete masks of dirty batches back into their base columns, on the device
        (sd_store_compact).  Rewritten batches number their live rows from 0; fully deleted batches leave the store."""
        nb = len(buckets or ())
        b = (C.c_int32 * max(1, nb))(*(buckets or ()))
        out = (C.c_int64 * 4)()
        self.api.check(self.api.lib.sd_store_compact(self.h, b if nb else None, nb, float(min_dirty_fraction), out))
        return dict(zip(("batches_rewritten", "batches_removed", "rows_purged", "bytes_written"), (int(x) for x in out)))

    def reclaim(self, max_live_fraction: float = 0.0) -> Dict[str, int]:
        """Give back the device memory of superseded batch versions (sd_store_reclaim): slabs nothing live lies in are
        freed, slabs at most `max_live_fraction` live are emptied into fresh ones first.  Slabs an unfinished scan can
        still read are deferred to a later call."""
        out = (C.c_int64 * 4)()
        self.api.check(self.api.lib.sd_store_reclaim(self.h, float(max_live_fraction), out))
        return dict(zip(("slabs_freed", "bytes_freed", "bytes_moved", "slabs_deferred"), (int(x) for x in out)))

    def extent_bytes(self):
        """(bytes of the current batch versions' allocations, bytes only replaced versions kept for open scans hold)."""
        out = (C.c_int64 * 2)()
        self.api.check(self.api.lib.sdx_store_extent_bytes(self.h, out))
        return int(out[0]), int(out[1])

    def get_deletes(self, batch_index: int) -> bytes:
        """A batch's delete mask [0][numBaseRows][numDeletes][positions] (sdx_store_get_deletes)."""
        ln = C.c_int64()
        rc = self.api.lib.sdx_store_get_deletes(self.h, batch_index, None, 0, C.byref(ln))
        if rc not in (0, SD_ERR_OVERFLOW):
            self.api.check(rc)
        buf = C.create_string_buffer(max(1, ln.value))
        self.api.check(self.api.lib.sdx_store_get_deletes(self.h, batch_index, buf, len(buf), C.byref(ln)))
        return buf.raw[: ln.value]


def last_mutation_timing(api: Api) -> Dict[str, float]:
    """Device and host times of the calling thread's last UPDATE / DELETE (sdx_last_mutation_timing)."""
    out = (C.c_double * 6)()
    api.check(api.lib.sdx_last_mutation_timing(out))
    return dict(zip(("scan_ms", "sort_ms", "merge_ms", "install_ms", "statement_ms", "rows"), list(out)))


def last_compaction_timing(api: Api) -> Dict[str, float]:
    """Device and host times of the calling thread's last compaction (sdx_last_compaction_timing)."""
    out = (C.c_double * 6)()
    api.check(api.lib.sdx_last_compaction_timing(out))
    return dict(zip(("materialise_ms", "encode_ms", "host_ms", "compaction_ms", "rows_read", "bytes_read"), list(out)))


def last_reclaim_timing(api: Api) -> Dict[str, float]:
    """Host and device times of the calling thread's last reclaim (sdx_last_reclaim_timing)."""
    out = (C.c_double * 6)()
    api.check(api.lib.sdx_last_reclaim_timing(out))
    return dict(zip(("plan_ms", "copy_ms", "install_ms", "free_ms", "reclaim_ms", "rounds"), list(out)))


def image_width(api: Api, dict_image: bool, elem_bytes: int, ndistinct: int = 0, lo: int = 0, hi: int = 0) -> int:
    """Width in bytes (0: none) of the scan image the store builds for one column of one batch (sdx_image_width)."""
    w = C.c_int32()
    api.check(api.lib.sdx_image_width(1 if dict_image else 0, elem_bytes, ndistinct, lo, hi, C.byref(w)))
    return w.value
