// sd_device.h -- structures shared by the host engine and the device kernels.
// Self-contained (no std headers) so that the NVRTC-compiled plan kernels can include it as text.
#ifndef SD_DEVICE_H
#define SD_DEVICE_H

#ifdef __CUDACC_RTC__
typedef signed char int8_t;
typedef unsigned char uint8_t;
typedef short int16_t;
typedef unsigned short uint16_t;
typedef int int32_t;
typedef unsigned int uint32_t;
typedef long long int64_t;
typedef unsigned long long uint64_t;
typedef unsigned long long uintptr_t;
#else
#include <stdint.h>
#endif

namespace sd {

// ---- column encodings as the kernels see them (enc/ColumnEncoding.scala:766-773) -------------
enum : int32_t { ENC_UNCOMPRESSED = 0, ENC_RUN_LENGTH = 1, ENC_DICTIONARY = 2, ENC_BIG_DICTIONARY = 3, ENC_BOOLEAN_BITSET = 4,
                 // engine-internal view of an Uncompressed variable-width STRING body (back-to-back [len:int32][bytes]
                 // records, enc/Uncompressed.scala:116-161): DevCol.data = int32 byte position of every stored value's record
                 // (built once at upload by walking the sequential cursor), DevCol.dict = the body the positions point into
                 ENC_STR_RAW = 5 };

// ---- register value kinds of a scan column ---------------------------------------------------
// K_CODE: a STRING column travels through the kernel as a 32-bit reference.  Dictionary-encoded batches: the per-batch
// dictionary index ("code"); predicates on it are per-batch truth tables and group keys per-batch code->group maps,
// both prepared on the host from the (tiny) dictionaries -- the reference's own dictionary-array shortcut
// (SnappyHashAggregateExec.scala:1340-1369) taken to its conclusion.  Uncompressed variable-width batches
// (ENC_STR_RAW): the byte position of the value's [len][bytes] record; predicates compare the bytes on the device and
// hash-table keys are compared / hashed by their bytes.  Which of the two a batch uses is uniform per (batch, column).
enum : int32_t { K_I8 = 0, K_I16 = 1, K_I32 = 2, K_I64 = 3, K_F32 = 4, K_F64 = 5, K_BOOL = 6, K_CODE = 7 };

// ---- tiling ----------------------------------------------------------------------------------
// A CTA of THREADS threads processes tiles of THREADS*RPT rows (RPT = rows per thread per tile, a per-plan
// tunable: 2, 4 or 8); thread t owns the row pairs tile + u*2*THREADS + 2*t + {0,1}, u < RPT/2, so that
// every per-column load instruction is a fully coalesced 16/8/4/2-byte-per-lane vector load.  A work item
// ("chunk") is CHUNK_ROWS rows of one batch.
constexpr int THREADS = 256;
constexpr int CHUNK_ROWS = 8192;
constexpr int NULL_PREFIX_ROWS = 512;         // granularity of the host-computed "nulls before" prefix
constexpr int NULL_PREFIX_WORDS = NULL_PREFIX_ROWS / 64;
constexpr int MAX_RPT = 8;

// bytes one row of a column occupies in a stage of the shared-memory ring (K_CODE: room for int32 indexes)
constexpr int kind_stage_width(int k) { return (k == K_I64 || k == K_F64) ? 8 : (k == K_I32 || k == K_F32 || k == K_CODE) ? 4 : (k == K_I16) ? 2 : 1; }
constexpr int MAX_STAGES = 12;
constexpr int MAX_SCAN_COLS = 64;   // scan columns of one fused plan
constexpr int RING_ALIGN_SLACK = 128;   // shared memory reserved to start the ring on a 128-byte boundary (sd_kernels.cuh)

// bytes of TileSmem<PLAN> for a plan with nc scan columns (kept in sync with sd_kernels.cuh)
constexpr int tile_smem_bytes(int nc, int rpt) {
  return (THREADS * rpt / 32) * 4 + (nc > 0 ? nc : 1) * ((THREADS * rpt / 32) * 4 + (THREADS * rpt / 64) * 4 + 16) + 8 +
         (THREADS / 32) * 4 + (nc > 0 ? nc : 1) * (THREADS / 32) * 2 * 4;   // per-warp cursors of the overlay path
}

constexpr int MAX_LITERALS = 64;
constexpr int MAX_TABLES = 40;   // per-batch lookup tables (truth tables + key maps) of one plan
constexpr int MAX_KEYS = 4;        // dense group table (MODE_GROUPS): mixed-radix index over <= 4 dictionary keys
constexpr int MAX_HASH_KEYS = 32;  // hash table (MODE_HASH): one NULL bit per key in a 32-bit word
constexpr int ROLLUP_MAX_SHIFTS = 16;   // grouping sets: moment / covariance shifts the roll-up re-centres (sd_rollup.cu)

// One update delta of one column (enc/ColumnDeltaEncoder.scala:300-331): ascending positions +
// values in the column's normal encoding; null bits index the relative entry.
struct DevDelta {
  const int32_t* positions;   // [n] ascending base-row ordinals
  const uint8_t* data;        // first encoded value / index
  const uint64_t* nulls;      // relative null words (8-byte aligned copy) or nullptr
  const uint8_t* dict;        // int32/int64 dictionary values (ENC_DICTIONARY of INT/LONG) or code map
  int32_t n;
  int32_t nwords;
  int32_t enc;
  int32_t dict_n;
};

// One scan column of one batch.
struct DevCol {
  const uint8_t* data;        // first encoded value (uncompressed), first index (dictionary),
                              // first word (bitset) or first run (run length); 128-byte aligned
  const uint64_t* nulls;      // null words (8-byte aligned copy), or nullptr when the batch has none
  const int32_t* tile_nulls;  // [ceil(rows/512) + 1] nulls before row 512*k (last entry: all nulls), or nullptr
  const uint8_t* dict;        // int32/int64 dictionary values; for RLE strings: int32 code per run
  const int32_t* run_ends;    // RLE: [nruns] exclusive end (in stored-value index) of each run
  const DevDelta* delta0;     // depth-0 delta (wins on equal position) or nullptr
  const DevDelta* delta1;     // depth-1 delta or nullptr
  int32_t nwords;             // number of null words (trailing zero words are trimmed)
  int32_t enc;
  int32_t dict_n;             // dictionary entries (NULL code == dict_n for nullable columns)
  int32_t nruns;
  // scan image (sd_image.cu): the same values as `data`, narrower, built and verified on the device when the batch version
  // was created; only the staged loads read it.  Floating-point kinds: 1-byte indexes into img_tab, the distinct bit
  // patterns (<= IMG_DICT_MAX).  Integral kinds and dictionary codes: unsigned offsets from img_tab[0] (frame of reference).
  const uint8_t* img;         // img_w bytes per row, 128-byte aligned, or nullptr
  const uint64_t* img_tab;
  int32_t img_w;              // 1 or 2
  int32_t img_n;              // words of img_tab (dictionary entries; 1 for a frame of reference)
};

constexpr int IMG_DICT_MAX = 256;
// words of the scan kernel's per-chunk shared-memory copy of a column's img_tab
constexpr int img_smem_words(int k) { return (k == K_F64 || k == K_F32) ? IMG_DICT_MAX : (k == K_BOOL || k == K_I8) ? 0 : 1; }

template <int NC>
struct DevBatch {
  int32_t num_rows;
  int32_t num_deletes;
  const int32_t* deletes;     // ascending deleted ordinals or nullptr (enc/ColumnDeleteEncoder.scala:101-134)
  const uint8_t* aux;         // per-plan per-batch tables: key code->group maps, predicate truth tables
  int32_t flags;              // BATCH_ALL_FAST | BATCH_FAST_OVERLAY | BATCH_FAST_NULLS (0: general per-row decode)
  int32_t pad_;
  DevCol cols[NC > 0 ? NC : 1];
};
constexpr int32_t BATCH_ALL_FAST = 1;      // no nulls, simple encodings, no deltas, no deletes: staged vector loads only
constexpr int32_t BATCH_FAST_NULLS = 4;    // simple encodings, some columns have NULLs: the tile's stored (non-null) values are staged and
                                           // consumers map row -> value index through the null words
constexpr int32_t BATCH_FAST_OVERLAY = 2;  // base columns as above, plus update deltas and/or a delete mask: staged loads,
                                           // then the few updated / deleted rows of each tile are patched in registers

struct Literals {
  int64_t i[MAX_LITERALS];
  double d[MAX_LITERALS];
  uint64_t nullmask;          // bit k: literal slot k is NULL
};

// aggregation strategy of a generated plan struct
//   MODE_NOKEY  no grouping keys: accumulators in registers
//   MODE_GROUPS dictionary-STRING keys: dense [group][slot] table over query-global dictionary ids
//   MODE_HASH   general keys (integral / date / timestamp / boolean / dictionary codes, nullable): open-addressing
//               hash table in global memory (the role SHAMap / ByteBufferHashMap plays in the reference,
//               encoders/.../collection/ByteBufferHashMap.scala:136-187)
//   MODE_PROJECT no aggregate: rows that pass the filter are emitted as fixed-width records
//               [uint32 batch][uint32 null bits][8 bytes x NPROJ] (strings as dictionary codes; the host
//               turns records into UnsafeRows)
//   MODE_MUTATE  UPDATE / DELETE (SD_PLAN_MUTATE): every live row that passes the WHERE becomes a record
//               [uint64 batch << 32 | row][uint64 null bits][8 bytes x max(NPROJ, 1)] -- the first word is the
//               (batch, row) sort key of the merge that follows (sd_mutate.cu)
enum : int32_t { MODE_NOKEY = 0, MODE_GROUPS = 1, MODE_HASH = 2, MODE_PROJECT = 3, MODE_MUTATE = 4 };

// Device hash table of MODE_HASH: entry e = state[e] (0 empty, 1 being written, 2 full), keys[e][NK] (int64 codes),
// knull[e] (bit k: key k is NULL), vals[e][NSLOT].
struct HashTable {
  uint32_t* state;
  int64_t* keys;
  uint32_t* knull;
  uint64_t* vals;
  uint64_t* shifts;       // [capacity][NSHIFT] K words of moment aggregates (SHIFT_EMPTY when unclaimed), or nullptr
  uint32_t mask;          // capacity - 1 (capacity is a power of two)
  uint32_t max_probe;
  uint32_t* overflow;     // set to 1 when an insert gives up: the host grows the table and replays
  uint32_t* count;        // number of distinct keys inserted
};

// where the dense [group][slot] table of a MODE_GROUPS launch lives (chosen per launch from its size):
//   TABLE_PRIVATE        one private copy per thread in shared memory, no atomics (few groups: TPC-H Q1)
//   TABLE_SHARED_ATOMIC  one copy per CTA in shared memory, shared-memory atomics
//   TABLE_GLOBAL_ATOMIC  the running result in global memory, global atomics (RED.ADD.F64 is native)
//   TABLE_REGS           one private copy per thread in REGISTERS (predicated accumulators; kernel variant with
//                        PLAN::REG_GROUPS >= ngroups): leaves all shared memory to the staged ring
enum : int32_t { TABLE_PRIVATE = 0, TABLE_SHARED_ATOMIC = 1, TABLE_GLOBAL_ATOMIC = 2, TABLE_REGS = 3 };

// accumulator slot operations; every slot is 8 bytes
// SLOT_MIN_STR / SLOT_MAX_STR: the slot holds the device address of the winning value's [len][bytes] record (0: no value yet);
// values compare as unsigned bytes (MIN / MAX over STRING: the aggregate buffer is not fixed-width, which is what sends the
// reference down its ObjectHashSet path, SnappyHashAggregateExec.scala:82-94)
// SLOT_MIN_DEC / SLOT_MAX_DEC: the same for a DECIMAL wider than 18 digits, whose record is [len][big-endian two's-complement
// unscaled value]; records compare by their numeric value
// SLOT_FIRST / SLOT_LAST + SLOT_PAIR_VAL: one FIRST / LAST buffer, a pair of adjacent slots at an even slot index (16-byte
// aligned in every table: the plan's slot count is even too).  Word 0 is the order key of the row the pair holds, word 1 that
// row's value, stored as MIN / MAX store one (int64, double bits, or the address of a STRING / wide-DECIMAL record).  The pair
// combines as one unit: the smaller key (FIRST) or the larger key (LAST) wins and the value travels with it.
enum : int32_t { SLOT_ADD_F64 = 0, SLOT_ADD_I64 = 1, SLOT_MIN_I64 = 2, SLOT_MAX_I64 = 3, SLOT_MIN_F64 = 4, SLOT_MAX_F64 = 5,
                 SLOT_MIN_STR = 6, SLOT_MAX_STR = 7, SLOT_MIN_DEC = 8, SLOT_MAX_DEC = 9,
                 SLOT_FIRST = 10, SLOT_LAST = 11, SLOT_PAIR_VAL = 12 };
// Order key of a row: ((execution-wide batch sequence + 1) << 32) | (row ordinal << 1) | (1 when the value is NULL).  Unique per
// row of one execution and increasing in scan order across all its launches (and the same in a launch's replays).  An empty
// pair holds ORDER_EMPTY_FIRST (FIRST) or 0 (LAST): no row's key takes either, and every row's key beats them.
constexpr uint64_t ORDER_EMPTY_FIRST = 0xffffffffffffffffull;
constexpr bool is_order_op(int op) { return op == SLOT_FIRST || op == SLOT_LAST; }
// initial word of a slot (slot_identity of sd_kernels.cuh, plus the FIRST / LAST order keys), for host and device
constexpr uint64_t slot_initial(int op) {
  return op == SLOT_MIN_I64 ? 0x7fffffffffffffffull : op == SLOT_MAX_I64 ? 0x8000000000000000ull
       : op == SLOT_MIN_F64 ? 0x7ff8000000000000ull : op == SLOT_MAX_F64 ? 0xfff0000000000000ull
       : op == SLOT_FIRST ? ORDER_EMPTY_FIRST : 0ull;
}

// Moment aggregates (STDDEV / VARIANCE / SKEWNESS / KURTOSIS) sum S_j = sum (x - K)^j around one shift K per group and input.
// The K words are not slots: they live beside the running result ([ngroups][NSHIFT] after its [ngroups][NSLOT] entries) and
// beside the hash entries (HashTable.shifts), never in per-thread / per-CTA tables or partials.  A K word is SHIFT_EMPTY until
// the group's first non-null input claims it with a set-once CAS; every contribution of one execution uses that K, so the sums
// stay plain commutative additions.  SHIFT_EMPTY is all ones (a byte memset sets it): a NaN no input reaches, because NaN
// inputs claim the canonical NaN 0x7ff8000000000000.
constexpr uint64_t SHIFT_EMPTY = 0xffffffffffffffffull;

struct ScanArgs {
  const void* batches;            // DevBatch<NC>[nbatches]
  const int32_t* chunk_prefix;    // [nbatches + 1] cumulative chunk counts
  int32_t nbatches;
  int32_t total_chunks;
  uint64_t* partials;             // [gridDim.x][ngroups * NSLOT] per-CTA partial tables
  uint64_t* result;               // [ngroups * NSLOT] running result (combined into, not overwritten)
  uint64_t* shifts;               // moment aggregates: [ngroups][NSHIFT] K words (SHIFT_EMPTY until claimed), else nullptr
  unsigned int* ticket;           // CTA completion counter (reset by the last CTA)
  unsigned long long* counters;   // [0] rows scanned, [1] rows that passed the filter
  int32_t ngroups;                // group slots of the dense group table (1 without keys)
  int32_t table_mode;             // TABLE_PRIVATE | TABLE_SHARED_ATOMIC | TABLE_GLOBAL_ATOMIC
  int32_t ring_off;               // byte offset of [mbarriers][stage ring] in dynamic shared memory
  int32_t nstages;                // stages of the ring actually allocated (<= MAX_STAGES)
  HashTable hash;                 // MODE_HASH
  int32_t radix[MAX_KEYS];        // group index = ((g0 * radix[1] + g1) * radix[2] + g2) ...
  // projection mode
  uint8_t* out_rows;              // MODE_PROJECT: output records
  unsigned long long* out_count;  // MODE_PROJECT: records produced (may exceed out_cap: the host grows and replays)
  int64_t out_cap;                // MODE_PROJECT: capacity in records
  int32_t batch_base;             // ordinal of this launch's first batch within the execution (MODE_PROJECT / MODE_MUTATE records;
                                  // the order keys of FIRST / LAST)
  int32_t chunk_rows;             // rows per work item (multiple of every tile size; default CHUNK_ROWS)
  const uint8_t* lit_pool;        // bytes of the STRING literals of this execution (literal slot k: lits.i[k] = offset << 32 | length);
                                  // a wide DECIMAL literal is its 16-byte little-endian unscaled value there, 16-byte aligned
  int32_t fresh;                  // 1: first launch of an execution -- the last CTA OVERWRITES `result` (no host-side
                                  // identity upload, one dependent operation less in front of the kernel)
  int32_t shift_cache_off;        // MODE_GROUPS with moment aggregates, TABLE_PRIVATE / TABLE_SHARED_ATOMIC: byte offset in
                                  // dynamic shared memory of the CTA's copy of the K words, [ngroups][NSHIFT]; -1: none
  int32_t img_off;                // byte offset in dynamic shared memory of the per-chunk copies of the columns' img_tab
                                  // (img_smem_words per column, or RingArgs.img_col); -1: the staged loads read the verbatim values
  Literals lits;
};
// Ring layout of a launch of a dense group-by's two-CTA kernel (sd_kernels.cuh scan_aggregate_kernel_2cta), sized by the
// widths the launch streams; every other kernel reads the verbatim layout as constants (stage_col_off / img_col_off)
struct RingArgs {
  int32_t stage_bytes;                    // bytes of one stage
  int32_t stage_off[MAX_SCAN_COLS];       // byte offset of column c's region in a stage (128-byte aligned)
  int32_t img_col[MAX_SCAN_COLS];         // word offset of column c's img_tab copy from ScanArgs.img_off
};
static_assert(sizeof(ScanArgs) + sizeof(RingArgs) <= 4096, "kernel parameters are limited to 4 KB");

}  // namespace sd
#endif
