/*
 * snappy_gpu.h -- C ABI of libsnappygpu.so, the H100-native replacement for the inside of
 * SnappyData's partial-aggregation stage:
 *
 *     ColumnTableScan -> [FilterExec / ProjectExec] -> SnappyHashAggregateExec(Partial)
 *
 * These entry points are what a JNI shim on the reference side binds (INTEGRATION.md shows it).
 * Plain pointers and sizes only; no C++ / torch types.  Every function returns 0 on success and a
 * non-zero sd_status otherwise; sd_last_error() then holds a thread-local message.  There is NO
 * CPU fallback: a plan or buffer the GPU path cannot execute is an error (the reference's
 * CodegenSparkFallback, core/.../execution/CodegenSparkFallback.scala:48-134, is deliberately not
 * mirrored; BASELINE.json north_star).
 *
 * Citations are to /root/reference; enc = encoders/src/main/scala/org/apache/spark/sql/execution/
 * columnar/encoding, core = core/src/main/scala/org/apache/spark/sql.
 *
 * Threading (SURVEY.md 8b): one thread drives one sd_plan from create to destroy; distinct plans may
 * be driven concurrently from distinct threads; an sd_store may be shared by plans (reads only while
 * plans scan it).
 */
#ifndef SNAPPY_GPU_H
#define SNAPPY_GPU_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SD_ABI_VERSION 2

typedef enum sd_status {
  SD_OK = 0,
  SD_ERR_INVALID = 1,      /* malformed descriptor / buffer                         */
  SD_ERR_UNSUPPORTED = 2,  /* plan shape or encoding the GPU path does not execute  */
  SD_ERR_CUDA = 3,         /* CUDA runtime / driver / NVRTC failure                 */
  SD_ERR_OVERFLOW = 4,     /* caller's output buffer too small (outLen = needed)    */
  SD_ERR_STATE = 5         /* call sequence violation                               */
} sd_status;

/* SQL types of scan columns / expression nodes (Catalyst DataType of the attribute;
 * core/execution/columnar/ColumnTableScan.scala:684-760 picks the decoder read method from it). */
typedef enum sd_type {
  SD_BOOLEAN = 1, SD_BYTE = 2, SD_SHORT = 3, SD_INT = 4, SD_LONG = 5, SD_FLOAT = 6, SD_DOUBLE = 7,
  SD_DATE = 8,       /* int32 days since epoch       */
  SD_TIMESTAMP = 9,  /* int64 microseconds           */
  SD_STRING = 10,    /* UTF8String                   */
  SD_DECIMAL = 11    /* column values: precision <= 18, int64 unscaled (enc/Uncompressed.scala:95-98); precision 19..38,
                        back-to-back [int32 len][BigInteger.toByteArray() of the unscaled value, 1..16 bytes]
                        (enc/Uncompressed.scala:330-345).  A "wide" DECIMAL (precision > 18) is read, compared, cast up,
                        tested with IN / IS [NOT] NULL, grouped and aggregated; arithmetic on it, casts from it to anything
                        but an equal or wider DECIMAL, startsWith and SET values of that type are SD_ERR_UNSUPPORTED; it is
                        refused in update deltas, sd_store_encode_batch and sd_store_compact.  Aggregate buffers / results
                        may be wider (SUM: DECIMAL(min(38,p+10),s)), see sd_agg */
} sd_type;

/* One projected scan column (ColumnTableScan.output attribute). */
typedef struct sd_column {
  int32_t type;           /* sd_type                                                  */
  int32_t nullable;       /* field.nullable: selects Nullable vs NotNull decoder
                             (enc/ColumnEncoding.scala:817-822)                       */
  int32_t table_ordinal;  /* 0-based column of the table (ColumnFormatKey.columnIndex-1) */
  int32_t scale;          /* SD_DECIMAL scale; else 0                                 */
  int32_t precision;      /* SD_DECIMAL precision (1..38 for a scan column); else 0   */
} sd_column;

/* Expression tree, flattened; children always precede parents.  Mirrors the Catalyst trees that
 * FilterExec / ProjectExec / the aggregate functions' children hold (SURVEY.md 8a a12, a16).
 * Semantics restated from Spark 2.1.1 (SURVEY.md Appendix B): SQL three-valued logic, NULL in any
 * operand of arithmetic/comparison => NULL, x / 0 => NULL, integral arithmetic wraps,
 * FLOAT/DOUBLE comparisons use the NaN-safe total order (NaN == NaN, NaN greatest, -0.0 == 0.0),
 * strings compare as unsigned bytes. */
typedef enum sd_op {
  SD_OP_COL = 1,        /* a = index into sd_plan_desc.cols                      */
  SD_OP_LIT = 2,        /* a = literal slot (runtime value, cf. ParamLiteral,
                           core/catalyst/expressions/ParamLiteral.scala:43-110)  */
  SD_OP_ADD = 10, SD_OP_SUB = 11, SD_OP_MUL = 12, SD_OP_DIV = 13, SD_OP_NEG = 14,
  SD_OP_CAST = 15,      /* a -> node type                                        */
  SD_OP_EQ = 20, SD_OP_NE = 21, SD_OP_LT = 22, SD_OP_LE = 23, SD_OP_GT = 24, SD_OP_GE = 25,
  SD_OP_AND = 30, SD_OP_OR = 31, SD_OP_NOT = 32,
  SD_OP_ISNULL = 33, SD_OP_ISNOTNULL = 34,
  SD_OP_IN = 35,        /* a = expr, b = first literal slot, c = number of literals */
  SD_OP_STARTSWITH = 36, /* a = string expr, b = literal node                    */
  SD_OP_PAIR = 37,      /* a = x node, b = y node, both DOUBLE; type DOUBLE, NULL when either is NULL.  Only as the input
                           of a two-input aggregate (COVAR_POP / COVAR_SAMP / CORR); anywhere else SD_ERR_INVALID */
  SD_OP_GROUPING_SET = 38, /* type SD_INT, a = one grouping-set mask.  Only as a member of a GROUPING_ID node's list */
  SD_OP_GROUPING_ID = 39   /* type SD_INT, a = index of the first of b consecutive GROUPING_SET nodes; only as the LAST entry of
                              sd_plan_desc.keys (GROUP BY ... WITH ROLLUP / WITH CUBE / GROUPING SETS, see below) */
} sd_op;

typedef struct sd_expr {
  int32_t op;    /* sd_op                     */
  int32_t type;  /* sd_type of the result     */
  int32_t a, b, c;   /* SD_DECIMAL-typed LIT / CAST nodes: c = (precision << 8) | scale of the node's type (a COL node takes
                        them from its column, NEG from its child; DECIMAL literal values are unscaled at that scale) */
} sd_expr;
#define SD_DEC_PS(precision, scale) (((precision) << 8) | (scale))

/* CAST follows Spark 2.1.1 Cast for the pairs the GPU path executes; every other pair is SD_ERR_UNSUPPORTED:
 *   integral <-> integral (wraps), integral/fp -> fp, fp -> integral (Java (int)/(long): NaN -> 0, saturating),
 *   numeric -> BOOLEAN (v != 0), BOOLEAN -> numeric (1 / 0), DECIMAL(p,s) -> DOUBLE/FLOAT (unscaled / 10^s),
 *   integral -> DECIMAL(p,s) (v * 10^s, NULL when it does not fit p digits), DECIMAL(p1,s1) -> DECIMAL(p2,s2 >= s1)
 *   (rescale, NULL when it does not fit).  Casts involving STRING, DATE or TIMESTAMP (other than the identity),
 *   DECIMAL -> integral and down-scaling DECIMAL casts are refused. */

/* Aggregate functions (Spark DeclarativeAggregate, SURVEY.md Appendix B.1-4) and their partial
 * buffer fields, in the order SnappyHashAggregateExec lays them out
 * (core/execution/aggregate/SnappyHashAggregateExec.scala:174-210,456-471):
 *   COUNT_STAR / COUNT : [count LONG]
 *   SUM                : [sum LONG (integral input) | DOUBLE (float/double input)]   (nullable)
 *   AVG                : [sum DOUBLE, count LONG]
 *   MIN / MAX          : [value of the input type]                                   (nullable)
 * DECIMAL(p,s) input (Spark 2.1.1 Sum / Average): SUM buffer and result DECIMAL(p+10,s); AVG buffers
 * [sum DECIMAL(p+10,s), count LONG], result DECIMAL(p+4,s+4) = sum / count rounded HALF_UP.  In UnsafeRows a DECIMAL
 * of precision <= 18 is its unscaled int64 in the fixed slot; wider ones are (offset << 32 | size) + the
 * BigInteger two's-complement big-endian bytes in a 16-byte reserved region (UnsafeRowWriter.write(Decimal)).
 * Wide DECIMAL input (precision > 18): SUM / AVG sum each value as four 32-bit limbs (exact below 2^31 rows per execution),
 * a total of more than min(38, p+10) digits is NULL -- in partial rows such a total is written as 10^(buffer precision), a
 * value no in-range total reaches, and the merges keep it so (they add partial totals exactly); MIN / MAX keep the input type; AVG's result is
 * DECIMAL(min(38,p+4), min(38,s+4)) rounded HALF_UP, NULL when it does not fit.
 * Moment aggregates (Spark 2.1.1 CentralMomentAgg; stddev / variance are the SAMP forms).  The input node must be DOUBLE (Spark
 * casts any other numeric child to DOUBLE, an SD_OP_CAST node here), else SD_ERR_INVALID.  Buffers are non-nullable DOUBLEs,
 * 0.0 before any input, in aggBufferAttributes order:
 *   STDDEV_POP / STDDEV_SAMP / VAR_POP / VAR_SAMP : [n, avg, m2]
 *   SKEWNESS                                      : [n, avg, m2, m3]
 *   KURTOSIS                                      : [n, avg, m2, m3, m4]
 * (m_k = sum (x - avg)^k over the non-null inputs).  Merge is Spark's (Chan et al.):
 *   n = n1+n2, d = avg2-avg1, dN = n == 0 ? 0 : d/n, avg = avg1 + dN*n2, m2 = m2_1+m2_2 + d*dN*n1*n2,
 *   m3 = m3_1+m3_2 + dN^2*d*n1*n2*(n1-n2) + 3dN*(n1*m2_2 - n2*m2_1),
 *   m4 = m4_1+m4_2 + dN^3*d*n1*n2*(n1^2-n1*n2+n2^2) + 6dN^2*(n1^2*m2_2 + n2^2*m2_1) + 4dN*(n1*m3_2 - n2*m3_1).
 * Results are DOUBLE, NULL when n == 0; VAR_POP m2/n; VAR_SAMP NaN when n == 1, else m2/(n-1); STDDEV_* their square roots;
 * SKEWNESS NaN when m2 == 0, else sqrt(n)*m3/sqrt(m2^3); KURTOSIS NaN when m2 == 0, else n*m4/m2^2 - 3.  A NaN or +-Inf input
 * makes the group's results NaN.  The device sums (x - K)^j around one shift K per group and input (the first value the group
 * sees) and the partial rows carry the buffers above; plans with moment aggregates have no dense partials export
 * (sd_plan_partials_layout / sd_plan_export_partials / sd_plan_import_partials: SD_ERR_UNSUPPORTED).
 * Two-input aggregates (Spark 2.1.1 Covariance / Corr, restated from upstream Spark; the fork's source is not at hand).  The
 * input node must be an SD_OP_PAIR of two DOUBLE nodes (x, y), else SD_ERR_INVALID; a row counts only when both are non-null.
 * Buffers are non-nullable DOUBLEs, 0.0 before any input, in aggBufferAttributes order:
 *   COVAR_POP / COVAR_SAMP : [n, xAvg, yAvg, ck]
 *   CORR                   : [n, xAvg, yAvg, ck, xMk, yMk]
 * (ck = sum (x - xAvg)(y - yAvg), xMk = sum (x - xAvg)^2, yMk likewise).  Merge:
 *   n = n1+n2, dx = xAvg2-xAvg1, dxN = n == 0 ? 0 : dx/n, dy / dyN likewise, xAvg = xAvg1 + dxN*n2, yAvg = yAvg1 + dyN*n2,
 *   ck = ck1+ck2 + dx*dyN*n1*n2, xMk = xMk1+xMk2 + dx*dxN*n1*n2, yMk likewise.
 * Results are DOUBLE, NULL when n == 0; COVAR_POP ck/n; COVAR_SAMP NaN when n == 1, else ck/(n-1); CORR NaN when n == 1, else
 * ck/sqrt(xMk*yMk).  The device sums (x - Kx), (y - Ky), (x - Kx)(y - Ky) (and for CORR the squares) around one shift pair
 * (Kx, Ky) per group and input pair.  A group in which a counted row has a NaN or +-Inf x or y gets NaN in every buffer but n,
 * so its results are NaN (Spark's row-order update gives +-Inf or NaN there, depending on where the row falls).  Plans with
 * these aggregates have no dense partials export either.
 * Grouping sets (Spark 2.1.1 Expand under the partial aggregate for GROUP BY ... WITH ROLLUP / WITH CUBE / GROUPING SETS; the
 * analyzer rule ResolveGroupingAnalytics is restated from upstream Spark, the fork's source is not at hand).  The last key is an
 * SD_OP_GROUPING_ID node; the n keys before it are the GROUP BY expressions.  Each GROUPING_SET mask follows SnappyParser's
 * convention (core/SnappyParser.scala:564-571): bit (n-1-k) set <=> key k is absent from the set (NULL in its rows).  ROLLUP(k1..kn)
 * = masks (1 << i) - 1 for i = 0..n, CUBE = 0 .. 2^n - 1.  Partial rows are UnsafeRow(k1..kn, gid, aggregate buffers) and final
 * rows keys ++ gid ++ one value per aggregate, gid = the set's mask (INT, NOT NULL): a key absent from a set and a key NULL in the
 * data are different groups.  Aggregate inputs read the original values in every set; no input rows, no output rows (not even
 * for the () set).  sd_final_merge / sd_partial_merge treat gid as one more INT key.  The device scans once with the plain
 * GROUP BY k1..kn kernel and rolls its groups up into every set.  SD_ERR_INVALID: a GROUPING_SET node that is not in a
 * GROUPING_ID list; a GROUPING_ID node that is not the last key, or that is an operand, a filter, an aggregate input, a projection
 * or a SET value; a mask with bits at or above n; b < 1.  SD_ERR_UNSUPPORTED: duplicate masks; n == 0 (no GROUP BY expression
 * before the GROUPING_ID); n > 31; more than 4096 sets; more than 16 moment / covariance shifts (one per distinct moment input,
 * two per distinct PAIR); a GROUPING_ID in an SD_PLAN_MUTATE or projection plan.  These plans have no dense partials export.
 * FIRST / LAST (Spark 2.1.1 First / Last, restated from upstream Spark; SQL first / first_value / last / last_value, the _IGNORE_NULLS
 * codes for ignoreNulls = true).  Any input type; a STRING input and a DECIMAL input wider than 18 digits must be a column
 * (else SD_ERR_UNSUPPORTED).  Buffers, in aggBufferAttributes order: [value of the input type (nullable), valueSet BOOLEAN],
 * [NULL, false] before any input.  Update, in scan order: FIRST value = valueSet ? value : x, LAST value = x, then valueSet = true;
 * with ignoreNulls only rows whose x is not NULL count.  Rows the filter rejects and deleted rows do not count; an updated row
 * counts with its current value.  Scan order of one execution: batches in the order the engine receives them (sd_batch_submit
 * calls and the row-buffer batch of sd_rows_submit in call order, a store scan in its snapshot's batch order), rows of a batch
 * in ordinal order.  Merge of partial rows, in the order they are given (sd_partial_merge / sd_final_merge; sd_plan_exchange
 * merges the ranks in rank order): FIRST value = valueSet1 ? value1 : value2, LAST value = valueSet2 ? value2 : value1,
 * valueSet = valueSet1 || valueSet2.  The result is value.  The device keeps per group the row with the smallest (FIRST) or
 * largest (LAST) scan position, whatever order its CTAs run in.  These plans have no dense partials export.  A scan of a batch
 * whose update delta holds a STRING that the batch's dictionary lacks, under FIRST / LAST of that column, is SD_ERR_UNSUPPORTED
 * (such a string has no device record; sd_store_compact folds it into the dictionary). */
typedef enum sd_agg_fn {
  SD_AGG_COUNT_STAR = 1, SD_AGG_COUNT = 2, SD_AGG_SUM = 3, SD_AGG_AVG = 4, SD_AGG_MIN = 5, SD_AGG_MAX = 6,
  SD_AGG_STDDEV_POP = 7, SD_AGG_STDDEV_SAMP = 8, SD_AGG_VAR_POP = 9, SD_AGG_VAR_SAMP = 10, SD_AGG_SKEWNESS = 11,
  SD_AGG_KURTOSIS = 12, SD_AGG_COVAR_POP = 13, SD_AGG_COVAR_SAMP = 14, SD_AGG_CORR = 15,
  SD_AGG_FIRST = 16, SD_AGG_LAST = 17, SD_AGG_FIRST_IGNORE_NULLS = 18, SD_AGG_LAST_IGNORE_NULLS = 19
} sd_agg_fn;

typedef struct sd_agg {
  int32_t fn;    /* sd_agg_fn                               */
  int32_t expr;  /* input expression node; -1 for COUNT(*)  */
} sd_agg;

/* The fused plan: scan columns -> filter -> (group keys, aggregates) | projection. */
typedef struct sd_plan_desc {
  int32_t abi_version;          /* SD_ABI_VERSION                                        */
  int32_t ncols;   const sd_column* cols;
  int32_t nexprs;  const sd_expr* exprs;
  int32_t filter;               /* root node of the FilterExec condition, or -1          */
  int32_t nkeys;   const int32_t* keys;    /* grouping expressions (node indexes)        */
  int32_t naggs;   const sd_agg* aggs;
  int32_t nproj;   const int32_t* proj;    /* naggs == 0 && nkeys == 0: output columns   */
  int32_t nliterals; const int32_t* literal_types;   /* sd_type per literal slot         */
  int32_t flags;                /* 0, or SD_PLAN_MUTATE                                  */
} sd_plan_desc;

/* An UPDATE / DELETE over a resident store (sd_plan_update_store / sd_plan_delete_store).  No keys, no aggregates; `filter` is
 * the WHERE clause (-1: every live row); UPDATE: proj[i] is the value of the i-th SET target; DELETE: nproj = 0. */
#define SD_PLAN_MUTATE 1

typedef struct sd_literal {
  int32_t type;      /* sd_type                              */
  int32_t is_null;
  int64_t i;         /* integral / date / timestamp / boolean / decimal-unscaled value (ignored for a DECIMAL slot
                        of precision > 18, whose unscaled value is BigInteger.toByteArray() bytes in s / slen) */
  double  d;         /* FLOAT / DOUBLE value                 */
  const char* s;     /* STRING bytes (not NUL terminated)    */
  int32_t slen;
  int32_t pad_;
} sd_literal;

/* One column batch as ColumnBatchIterator serves it to the generated loop
 * (core/execution/columnar/ColumnBatchIterator.scala:53-231): per projected column the value
 * buffer (getColumnLob) and up to two update deltas (getUpdatedColumnDecoder, depth 0 and 1), the
 * delete mask (getDeletedColumnDecoder), the stats row (next()), ids.  Arrays are indexed like
 * sd_plan_desc.cols.  Buffers may be heap or direct memory; the library has finished reading (or
 * copied) them when sd_batch_submit returns (ownership rule, SURVEY.md 8b).  A buffer whose first
 * int32 is negative is a compressed envelope (encoders/.../store/CompressionUtils.scala:53-61): LZ4 (-1)
 * envelopes are accepted -- only the compressed bytes are copied and the block is expanded on the device (run-length
 * and variable-width STRING bodies, whose layout needs a host walk, are expanded on the host instead); Snappy (-2)
 * envelopes, compressed update deltas and compressed delete masks are decompressed on the host, as the reference's own
 * iterator does (ColumnBatchIterator.scala:102-113). */
typedef struct sd_batch {
  int32_t num_rows;
  int32_t ncols;
  const void* const* col_bufs;  const int64_t* col_lens;
  const void* const* delta0;    const int64_t* delta0_lens;   /* may be NULL; entries may be NULL */
  const void* const* delta1;    const int64_t* delta1_lens;
  const void* delete_buf;       int64_t delete_len;           /* may be NULL                      */
  const void* stats_row;        int64_t stats_len;            /* may be NULL (no batch skipping)  */
  int32_t stats_ncols;          /* number of table columns described by the stats row            */
  int32_t bucket_id;
  int64_t batch_id;
} sd_batch;

typedef struct sd_plan sd_plan;
typedef struct sd_store sd_store;

/* ---- lifecycle -------------------------------------------------------------------------------- */
int sd_init(int device);                       /* bind the calling thread's plans to a GPU          */
int sd_device_count(int* out);
const char* sd_last_error(void);               /* thread-local, valid until the next failing call   */
const char* sd_version(void);

/* page-locked host memory for a binding's staging area (the JNI shim copies heap byte[]s into it, so that no Java array
 * is pinned while CUDA work is queued and host->device copies out of it are real asynchronous DMA) */
int sd_host_alloc(int64_t bytes, void** out);
void sd_host_free(void* p);
/* page-lock memory the caller already owns and keeps for a long time (the region's off-heap column buffers): copies out of
 * it become asynchronous DMA at link speed instead of the driver's staged pageable copies (bench.py: e2e_pageable_unretained
 * is ~4x below the pinned legs) */
int sd_host_register(void* p, int64_t bytes);
int sd_host_unregister(void* p);

/* ---- plan (one per Spark task / partition; ColumnTableScan.doProduce + SnappyHashAggregateExec
 *      doProduce/doConsume fused, core/.../ColumnTableScan.scala:186-672,
 *      core/.../aggregate/SnappyHashAggregateExec.scala:240-263) --------------------------------- */
int sd_plan_create(const sd_plan_desc* desc, sd_plan** out);
int sd_plan_set_literals(sd_plan* p, const sd_literal* vals, int32_t n);
/* scan one batch from host buffers (copied to the device inside the call) */
int sd_batch_submit(sd_plan* p, const sd_batch* b);
/* row-buffer rows of the hybrid scan (core/execution/row/RowFormatScanRDD.scala; consumed through the
 * same loop with batch size 1, ColumnTableScan.scala:572-588): nrows UnsafeRows of the plan's
 * scan columns, each prefixed by its int64 size */
int sd_rows_submit(sd_plan* p, const void* rows, int64_t len, int32_t nrows);
/* finish the partition: run what is pending, emit partial-aggregate rows (or projected rows) as
 * repeated [int64 sizeInBytes][UnsafeRow(group keys ++ aggregate buffers)].  On SD_ERR_OVERFLOW
 * *out_len is the size needed and the call may be repeated. */
int sd_plan_finish(sd_plan* p, void* out_rows, int64_t cap, int64_t* out_len, int64_t* out_nrows);
/* make the handle reusable for another execution of the same (cached) plan */
int sd_plan_reset(sd_plan* p);
/* SQLMetrics of the two operators (ColumnTableScan.scala:111-127, SnappyHashAggregateExec.scala:132-137):
 * [0] numOutputRows (aggregate) [1] numRowsBuffer [2] columnBatchesSeen [3] updatedColumnCount
 * [4] deletedBatchCount [5] columnBatchesSkipped [6] aggTime (device ns) [7] kernel launches
 * [8] rows scanned [9] algorithmic bytes scanned [10] host->device bytes [11] scan numOutputRows */
#define SD_NUM_METRICS 12
int sd_plan_metrics(sd_plan* p, int64_t out[SD_NUM_METRICS]);
/* options.  SD_OPT_RETAIN_BUFFERS = 1: the caller keeps every buffer passed to sd_batch_submit alive and
 * unchanged until sd_plan_finish returns (e.g. ref-counted direct ByteBuffers retained by the operator); host->device
 * copies are then queued without a per-batch synchronisation.  Default 0: the reference's ownership rule (buffers
 * may be released when sd_batch_submit returns, ColumnBatchIterator.scala:165-184). */
#define SD_OPT_RETAIN_BUFFERS 1
int sd_plan_set_option(sd_plan* p, int32_t option, int64_t value);
/* run the plan's kernels on a caller-owned CUDA stream (cudaStream_t as void*), e.g. torch's */
int sd_plan_set_stream(sd_plan* p, void* cuda_stream);
/* kernel variant actually selected for the plan ("aot:<signature>" | "jit:<signature>") */
const char* sd_plan_kernel_name(sd_plan* p);
void sd_plan_destroy(sd_plan* p);

/* ---- device-resident column store (residency policy of this engine; the reference keeps batches
 *      in region memory and faults them in per scan, ColumnBatchIterator.scala:179-223) ---------- */
/* schema = the table's columns in table order (ColumnFormatRelation.schema); type and nullability
 * select the decoders exactly as field.dataType / field.nullable do in the reference */
int sd_store_create(int device, int32_t ncols, const sd_column* schema, sd_store** out);
/* upload one batch; b->col_bufs is indexed by TABLE column here (ncols = table width; NULL entries
 * for columns never scanned); delta arrays likewise */
int sd_store_put_batch(sd_store* s, const sd_batch* b);
/* ---- ingest: ColumnBatch creation ON THE DEVICE (SURVEY.md 8f N2).  Raw column values of one batch (what the reference's
 *      generated insert loop feeds its ColumnEncoders row by row, core/.../columnar/ColumnInsertExec.scala:326-822) are copied to
 *      the device once and encoded there into the reference's column buffers -- Uncompressed / Dictionary (first-seen
 *      order, int16 -> int32 indexes at 32767 entries) / BooleanBitSet with trimmed null words, the default encoder choice
 *      of enc/ColumnEncoding.scala:837-844 -- plus the stats row (lower / upper bound, null count per column;
 *      ColumnInsertExec.scala:848-921).  The batch is resident and scannable when the call returns; its bytes are the ones
 *      snappydata_b200/column_format.py writes for the same values (sdx_store_get_buffer / sdx_store_get_stats read them
 *      back).  cols[c] describes TABLE column c (values == NULL: not materialised). ---------------------------------- */
typedef struct sd_raw_column {
  const void* values;        /* num_rows values: BOOLEAN / BYTE 1 byte, SHORT 2, INT / DATE / FLOAT 4, LONG / TIMESTAMP / DOUBLE /
                                DECIMAL (unscaled) 8; STRING: int32 offsets[num_rows + 1] into str_bytes                  */
  const uint8_t* str_bytes;  /* STRING: the values' bytes back to back                                                */
  const uint8_t* nulls;      /* optional, 1 byte per row, non-zero = NULL; must be NULL for a NOT NULL column          */
} sd_raw_column;
int sd_store_encode_batch(sd_store* s, int32_t num_rows, const sd_raw_column* cols, int32_t ncols,
                          int32_t bucket_id, int64_t batch_id);
/* ColumnDeltaEncoder.merge (enc/ColumnDeltaEncoder.scala:348-556), host only: the new update delta of a column merged with what
 * the table holds -- another delta (existing_is_delta = 1: union of positions, the new one wins on equal positions, result is a
 * delta) or the full column of num_rows rows (existing_is_delta = 0: the delta folded into the column, result is a column
 * buffer) -- re-encoded with the type's default encoder.  Either input may be a compressed envelope. */
int sd_delta_merge(const sd_column* column, const void* new_delta, int64_t new_len, const void* existing, int64_t existing_len,
                   int32_t existing_is_delta, int32_t num_rows, void* out, int64_t cap, int64_t* out_len);
int sd_store_num_batches(sd_store* s, int64_t* out);
int sd_store_bytes(sd_store* s, int64_t* out);
/* scan every resident batch of the given buckets (NULL/0 = all) with plan p: stats-row skipping on
 * the host, then the fused kernels over the resident bytes; results are collected by sd_plan_finish */
int sd_plan_scan_store(sd_plan* p, sd_store* s, const int32_t* bucket_ids, int32_t nbuckets);
void sd_store_destroy(sd_store* s);

/* ---- UPDATE / DELETE on the device (the reference's ColumnUpdateExec / ColumnDeleteExec, core/.../columnar/ColumnUpdateExec.scala,
 *      ColumnDeleteExec.scala, with the store-side merge of ColumnDelta.apply, encoders/.../impl/ColumnDelta.scala:64-222).
 *      p is an SD_PLAN_MUTATE plan.  The WHERE sees each row's current value (base, depth-1, then depth-0 delta); deleted rows
 *      are not touched; SET values are computed from the row as it was before the statement.  UPDATE: every touched (batch,
 *      target) gets a new depth-0 delta = ColumnDeltaEncoder.merge(new, existing depth 0) in the type's default encoding; the
 *      stats row is merged as ColumnDelta.mergeStats does.  DELETE: the positions are merged into the batch's delete mask; a
 *      batch whose every row is deleted is no longer scanned.  A statement works on the batches present when it starts; its
 *      new batch versions are installed together under the store's lock (a scan sees all of them or none); statements on one
 *      store are serialised; a failing statement installs nothing.  Superseded delta / mask bytes stay in the store's arena
 *      until the store is destroyed (sd_store_bytes counts them).  Refused: STRING / BOOLEAN targets (SD_ERR_UNSUPPORTED), a SET
 *      type other than the target's (SD_ERR_INVALID), a target not resident in a touched batch (SD_ERR_INVALID), NULL into a
 *      NOT NULL target (SD_ERR_INVALID), a plan without SD_PLAN_MUTATE (SD_ERR_STATE). ------------------------------------ */
int sd_plan_update_store(sd_plan* p, sd_store* s, const int32_t* bucket_ids, int32_t nbuckets, const sd_literal* lits, int32_t nlits,
                         const int32_t* target_cols, int64_t* rows_updated);
int sd_plan_delete_store(sd_plan* p, sd_store* s, const int32_t* bucket_ids, int32_t nbuckets, const sd_literal* lits, int32_t nlits,
                         int64_t* rows_deleted);

/* ---- compaction on the device: fold the update deltas and delete masks of resident batches back into their base columns.
 *      Rewrites the dirty resident batches of the given buckets (NULL/0 = all) without their update deltas and delete masks.
 *      A batch is dirty when it carries a delta or a delete mask.  It is selected when
 *        (deleted rows + delta entries of its resident columns, depth 0 and 1) >= min_dirty_fraction * num_rows;
 *      min_dirty_fraction = 0 selects every dirty batch.  A batch whose every row is deleted is removed from the store.
 *      Every column of a selected batch that has a delta is rewritten -- every resident column when the batch has a delete
 *      mask -- as the bytes sd_store_encode_batch writes for the batch's live rows with their current values, in their
 *      original order, in the type's default encoding; other columns keep their bytes.  Rewritten columns get the encoder's
 *      stats entries, the row count becomes the live rows.  The new version keeps bucket_id and batch_id, gets a new identity
 *      and has no deltas and no mask: its row ordinals are the live rows renumbered from 0, and later UPDATE / DELETE
 *      statements address those.  Serialised with UPDATE / DELETE; works on the batches present when it starts; everything
 *      is installed in one step under the store's lock (a scan sees all of it or none).  Superseded bytes stay in the arena
 *      until sd_store_reclaim frees them or the store is destroyed.  Refused with nothing installed: a column that must be rewritten but that the engine
 *      cannot decode -- an Uncompressed (variable-width) STRING column, a column the scan does not support --
 *      (SD_ERR_UNSUPPORTED, naming batch and column); a negative or NaN min_dirty_fraction, a null store (SD_ERR_INVALID).
 *      out[0] batches rewritten, out[1] batches removed, out[2] deleted rows purged, out[3] bytes written to the store's arena */
int sd_store_compact(sd_store* s, const int32_t* bucket_ids, int32_t nbuckets, double min_dirty_fraction, int64_t out[4]);

/* ---- reclaim: give back the device memory of superseded batch versions --------------------------------------------------
 *      UPDATE / DELETE / compaction leave every version they replace in the store's arena, because a scan of an older
 *      snapshot may still read it.  This call frees what no open scan can read.  Live bytes are the allocations of every
 *      current batch version plus those of replaced versions that an open scan may still read; a scan is open from its
 *      snapshot (sd_plan_scan_store) until its result is materialised (sd_plan_finish), sd_plan_reset or sd_plan_destroy.
 *      Every slab the store holds when the call starts is considered (the slab being allocated from is closed first, so
 *      max_live_fraction = 1 can empty every slab): a slab without live bytes is freed without copying; a slab whose live
 *      bytes are at most max_live_fraction x its size is evacuated -- the live bytes of current versions are copied on the
 *      device into fresh slabs of the same arena, emptiest slabs first, in rounds of at most one destination slab, and each
 *      round installs new versions of the batches it moved (same bytes, rows, bucket, batch id, stats, deltas and mask at
 *      new addresses, new identity) in one step under the store's lock.  A source slab an open scan can still read is
 *      deferred: a later call frees it.  0 only frees dead slabs; 1 repacks everything.  sd_store_bytes drops by the bytes
 *      that were allocated in the freed slabs.  Serialised with UPDATE / DELETE / compaction and the device encoder;
 *      sd_store_put_batch may run meanwhile.  A failing round installs and frees nothing (rounds already installed stay,
 *      their bytes identical; the error says so); a device pointer of a batch that lies in none of its recorded allocations
 *      fails the call before anything is copied (SD_ERR_STATE, naming batch and column); a null store or a NaN, negative or
 *      > 1 fraction is refused with nothing changed (SD_ERR_INVALID).
 *      out[0] slabs freed, out[1] slab bytes freed, out[2] bytes copied, out[3] slabs deferred */
int sd_store_reclaim(sd_store* s, double max_live_fraction, int64_t out[4]);

/* ---- final merge (SnappyHashAggregateExec(Final) / CollectAggregateExec.executeCollect,
 *      core/execution/aggregate/CollectAggregateExec.scala:67-121): merges partial rows of all
 *      partitions (sums add, counts add, min/max combine) and evaluates results (avg = sum/count).
 *      Host-side: payload is a handful of rows.  Output rows: keys ++ one result per aggregate. --- */
int sd_final_merge(const sd_plan_desc* desc, const void* partial_rows, int64_t len,
                   void* out_rows, int64_t cap, int64_t* out_len, int64_t* out_nrows);

/* the same merge reusing the analysis held by a plan handle (no per-call plan analysis) */
int sd_plan_final_merge(sd_plan* p, const void* partial_rows, int64_t len,
                        void* out_rows, int64_t cap, int64_t* out_len, int64_t* out_nrows);

/* partial rows of several partitions -> ONE merged set of partial rows (same schema; a combiner in front of the final
 * stage).  sd_plan_exchange uses it after gathering every rank's rows. */
int sd_partial_merge(const sd_plan_desc* desc, const void* partial_rows, int64_t len,
                     void* out_rows, int64_t cap, int64_t* out_len, int64_t* out_nrows);   /* host only */
int sd_plan_partial_merge(sd_plan* p, const void* partial_rows, int64_t len,
                          void* out_rows, int64_t cap, int64_t* out_len, int64_t* out_nrows);

/* ---- the cross-partition exchange (SURVEY.md 8e): partial -> Exchange -> final as SnappyStrategies plans it
 *      (core/.../SnappyStrategies.scala:566-604).  One partition (= one sd_plan on one GPU) per rank; the exchange is ONE
 *      ncclAllGather over NVLink of every rank's partial rows BY VALUE, merged on every rank.  NCCL is dlopen'ed
 *      (libnccl.so.2, or $SD_NCCL_LIB); the caller only transports the 128-byte unique id from rank 0 to the others
 *      (torch.distributed / Spark broadcast / any RPC). ------------------------------------------------------------ */
typedef struct sd_comm sd_comm;
#define SD_COMM_ID_BYTES 128
int sd_comm_unique_id(void* out_id);                         /* rank 0 */
int sd_comm_create(const void* id, int32_t rank, int32_t world, int32_t device, sd_comm** out);   /* collective */
void sd_comm_destroy(sd_comm* c);
/* [0] world [1] bytes per rank of the gather slot [2] all-gathers issued [3] times the slot had to grow */
int sd_comm_info(sd_comm* c, int64_t out[4]);
/* collective, after this execution's scans: gathers + merges; sd_plan_finish then returns the MERGED partial rows
 * (identical on every rank; any number of groups -- the gather slot grows in lock step on all ranks) */
int sd_plan_exchange(sd_plan* p, sd_comm* c);
/* one execution of a cached plan over a resident store in one call:
 * reset -> set_literals -> scan_store -> [exchange when comm != NULL] -> finish */
int sd_plan_execute_store(sd_plan* p, sd_store* s, const int32_t* bucket_ids, int32_t nbuckets,
                          const sd_literal* lits, int32_t nlits, sd_comm* comm,
                          void* out_rows, int64_t cap, int64_t* out_len, int64_t* out_nrows);

/* ---- export of the dense partial table for an on-device exchange (NCCL all-reduce over NVLink of
 *      per-GPU partials; SURVEY.md 8e).  Writes nslots int64/double words per group into dev_out
 *      (device pointer) on the plan's stream.  Only for plans without string/hash keys, and without moment aggregates
 *      (their shifted sums of different GPUs do not add). ---------------------------------------------------------- */
int sd_plan_partials_layout(sd_plan* p, int32_t* ngroups, int32_t* nslots, int32_t* slot_is_f64);
int sd_plan_export_partials(sd_plan* p, void* dev_out, int64_t cap_bytes);
int sd_plan_import_partials(sd_plan* p, const void* dev_in, int64_t bytes);

/* ---- synthetic lineitem tables generated on the device straight into a store (bench/test
 *      utility; byte-identical to snappydata_b200/lineitem.py; not part of the reference boundary) */
int sdx_store_gen_lineitem(sd_store* s, int64_t first_row, int64_t nrows, int32_t rows_per_batch,
                           int32_t nbuckets, uint64_t seed, int32_t column_mask);
/* copy a resident buffer back to the host (tests: device generator == host generator) */
int sdx_store_get_buffer(sd_store* s, int64_t batch_index, int32_t table_col, void* out, int64_t cap,
                         int64_t* out_len);
/* host LZ4 prefix decoder used to lay out compressed column buffers (test hook) */
int64_t sdx_lz4_decode_prefix(const void* src, int64_t src_len, void* dst, int64_t want);
/* host decompression of a stored envelope [-codecId][uncompressedLen][payload] (LZ4 = 1, Snappy = 2), as the engine
 * applies it to update deltas, delete masks and Snappy column buffers (test hook; no CUDA call) */
int sdx_decompress_envelope(const void* buf, int64_t len, void* out, int64_t cap, int64_t* out_len);
/* a resident update delta (depth 0 or 1) of a batch's table column in the reference's byte layout (enc/ColumnDeltaEncoder.scala:
 * 300-331); SD_ERR_INVALID when the column has none at that depth, SD_ERR_UNSUPPORTED for a dictionary / bit-set delta */
int sdx_store_get_delta(sd_store* s, int64_t batch_index, int32_t table_col, int32_t depth, void* out, int64_t cap,
                        int64_t* out_len);
/* the delete mask of a resident batch: [0][numBaseRows][numDeletes][positions] (enc/ColumnDeleteEncoder.scala:101-134);
 * SD_ERR_INVALID when the batch has none */
int sdx_store_get_deletes(sd_store* s, int64_t batch_index, void* out, int64_t cap, int64_t* out_len);
/* device and host times of the calling thread's last sd_plan_update_store / sd_plan_delete_store (tools/mutation_bench.py):
 * [0] scan kernels ms [1] sort ms [2] counting + writing merge ms [3] host install ms [4] whole statement ms (host clock) [5] rows */
int sdx_last_mutation_timing(double out[6]);
/* the calling thread's last sd_store_compact: [0] materialise ms [1] encode ms (device events) [2] host layout + install ms
 * [3] whole call ms (host clock) [4] rows of the rewritten batches [5] bytes read (columns, deltas, delete masks) */
int sdx_last_compaction_timing(double out[6]);
/* the calling thread's last sd_store_reclaim: [0] inventory + planning ms (host) [1] copy ms (device events) [2] install ms
 * (host) [3] free ms (host) [4] whole call ms (host clock) [5] rounds */
int sdx_last_reclaim_timing(double out[6]);
/* bytes in the device allocations of the store's current batch versions (out[0]) and of the replaced versions kept for open
 * scans that the current ones do not share (out[1]) */
int sdx_store_extent_bytes(sd_store* s, int64_t out[2]);
/* stats row (UnsafeRow) of a resident batch */
int sdx_store_get_stats(sd_store* s, int64_t batch_index, void* out, int64_t cap, int64_t* out_len);
int sdx_store_batch_info(sd_store* s, int64_t batch_index, int32_t* num_rows, int32_t* bucket_id,
                         int64_t* batch_id);
/* device memory held by a store: the bytes of its slabs, and how many of them the driver allocated as compressible (the
 * store asks for generic compression where the device reports support; the hardware then compresses those slabs between
 * L2 and DRAM, invisibly to kernels and copies).  Read only. */
int sdx_store_memory_info(sd_store* s, int64_t* compressible_bytes, int64_t* slab_bytes);
/* scan images of a store's current batch versions (narrow byte-aligned copies of NOT NULL columns that the scan kernel's
 * staged loads read instead of the verbatim values; built and verified on the device when a version is created):
 * out[0] arena bytes they take, out[1] (batch, column) images, out[2] images whose device verification failed since the
 * store was created (those columns keep the verbatim path), out[3] microseconds spent building images.  Read only. */
int sdx_store_image_info(sd_store* s, int64_t out[4]);
/* the image rule for one column of one batch (host only, no CUDA call): width in bytes (0: no image) of a dictionary image
 * (dict != 0: DOUBLE / FLOAT with `ndistinct` distinct bit patterns) or of a frame of reference over [lo, hi] (integral
 * values of elem_bytes 2, 4 or 8 bytes) */
int sdx_image_width(int32_t dict, int32_t elem_bytes, uint64_t ndistinct, int64_t lo, int64_t hi, int32_t* width);
/* the batch-skipping decision (ColumnTableScan.scala:820-963) of a plan's filter for one stats row: *pass = 0 when the
 * batch would be skipped.  Host only, no CUDA call (test hook: tests/test_stats_predicate.py compares it with the oracle). */
int sdx_stats_pass(const sd_plan_desc* desc, const sd_literal* lits, int32_t nlits, const void* stats,
                   int64_t stats_len, int32_t stats_ncols, int32_t num_rows, int32_t* pass);
/* what each kernel launch of a plan since its last sd_plan_reset ran: SDX_LAUNCH_WORDS int64 per launch, in launch order
 * (test hook: the engine picks the decode path, kernel shape and group-table placement per batch and per launch; this
 * reports the choice and changes nothing).  Word:
 *   [0] accumulator (SDX_ACC_*)   [1] 1: the kernel variant with the per-row decode / overlay paths ran   [2] 1: the variant
 *   with NULL literal flags ran   [3] stages of the shared-memory ring (0: direct loads)   [4] rows per tile
 *   [5] rows per work item   [6] grid (CTAs)   [7] groups of the dense table (1 without one)   [8..11] batches of the launch
 *   on the BATCH_ALL_FAST, BATCH_FAST_NULLS, BATCH_FAST_OVERLAY and general per-row paths   [12] SDX_REPLAY_*: why the launch
 *   repeats an earlier one of the execution   [13] batches   [14] work items   [15] bytes of column values the launch
 *   reads: scan images where the staged loads take them, verbatim element bytes elsewhere (NULL words, deltas and
 *   dictionaries not counted)
 * The first SDX_LAUNCH_LOG_MAX launches are kept.  *n = launches kept; min(cap, *n) records are written to out;
 * SD_ERR_OVERFLOW when cap < *n. */
#define SDX_LAUNCH_WORDS 16
#define SDX_LAUNCH_LOG_MAX 4096
enum { SDX_ACC_NOKEY = 0, SDX_ACC_PRIVATE = 1, SDX_ACC_SHARED_ATOMIC = 2, SDX_ACC_GLOBAL_ATOMIC = 3, SDX_ACC_HASH = 4,
       SDX_ACC_REGTABLE = 5, SDX_ACC_ROWS = 6 /* projection / UPDATE / DELETE records */ };
enum { SDX_REPLAY_NONE = 0,
       SDX_REPLAY_HASH_SWITCH = 1,   /* the dense group table was given up for the hash table: earlier launches re-run  */
       SDX_REPLAY_HASH_GROW = 2,     /* the hash table grew: every launch of the execution re-runs                      */
       SDX_REPLAY_ROWS_GROW = 3 };   /* the projection / UPDATE / DELETE record buffer grew: every launch re-runs       */
int sdx_plan_launch_log(sd_plan* p, int64_t* out, int32_t cap, int32_t* n);
/* the roll-up of a grouping-sets plan's last execution (test / bench hook; the launch log and sd_plan_metrics cover the scan
 * only): [0] roll-up device ms (CUDA events, re-runs included) [1] fine groups of the scan [2] coarse groups emitted
 * [3] roll-up launches (a re-run after the roll-up table overflowed counts again).  All 0 for other plans. */
int sdx_plan_rollup_info(sd_plan* p, double out[4]);
/* expand n raw LZ4 blocks with the engine's device kernel (bench/test hook used by tools/lz4_bench.py): uploads the
 * blocks, places output i at a 16-byte boundary + dst_misalign, runs `reps` launches timed with CUDA events
 * (ms_per_launch = their mean) and copies output i to outs[i] when outs != NULL.  `dense` selects the kernel variant:
 * bit 0 = the denser shape (SD_TUNE_LZ4_DENSE), bit 1 = the window parse (SD_TUNE_LZ4_PARSE).  A corrupt block ->
 * SD_ERR_INVALID. */
int sdx_lz4_expand(int32_t device, const void* const* blocks, const int64_t* block_lens, const int64_t* out_lens,
                   int32_t n, int32_t dst_misalign, int32_t dense, int32_t reps, void* const* outs,
                   double* ms_per_launch);

#ifdef __cplusplus
}
#endif
#endif /* SNAPPY_GPU_H */
