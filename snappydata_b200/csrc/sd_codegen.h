// sd_codegen.h -- plan analysis and generation of the per-plan PLAN struct for sd_kernels.cuh.
#ifndef SD_CODEGEN_H
#define SD_CODEGEN_H

#include <string>
#include <vector>

#include "../../include/snappy_gpu.h"
#include "sd_device.h"

namespace sd {

// TABLE_KEYPTR: per dictionary code the device address (int64) of the entry's [len][bytes] record -- string keys of the
// hash table are held by reference and compared by their bytes
enum TableKind { TABLE_TRUTH = 0, TABLE_KEYMAP = 1, TABLE_KEYPTR = 2 };

// A per-batch lookup table indexed by a STRING column's dictionary code.
struct TableSpec {
  int kind;   // TableKind
  int col;    // scan column
  int node;   // TABLE_TRUTH: the predicate node evaluated per dictionary entry
  int key;    // TABLE_KEYMAP: index into keys
};

// GATE_VALUE_HI32 / GATE_VALUE_LO32: the two halves of a wide (128-bit) integer sum: v = (v >> 32) * 2^32 + (v & 0xffffffff);
// each half is summed in its own int64 slot (exact for < 2^31 rows per execution), recombined on the host
// GATE_STRREF: the value is a STRING column held by reference (address of its record; SlotSpec.table = its TABLE_KEYPTR table)
// GATE_LIMB0..3: the four 32-bit limbs of a wide DECIMAL (precision > 18) value v = l3 * 2^96 + l2 * 2^64 + l1 * 2^32 + l0
// (l0..l2 unsigned, l3 signed); each summed in its own int64 slot (exact for < 2^31 rows per execution), recombined on the host
// GATE_DECREF: the value is a wide DECIMAL column held by reference (address of its [len][bytes] record)
// GATE_POW1..4: S_j = sum (x - K)^j of a moment aggregate's input (the row leaves its candidate K, x, in S_1;
// sd_kernels.cuh apply_shifts fills them all once the group's K is known)
// GATE_PAIR_X / GATE_PAIR_Y: S_x = sum (x - Kx), S_y = sum (y - Ky) of a two-input aggregate's SD_OP_PAIR node (the row leaves
// its candidate Kx / Ky there, SHIFT_EMPTY when x or y is NULL); GATE_PAIR_XY: S_xy = sum (x - Kx)(y - Ky); GATE_PAIR_XX /
// GATE_PAIR_YY: CORR's sum (x - Kx)^2 / sum (y - Ky)^2.  apply_shifts fills them like the moment sums
// GATE_ORDER_KEY / GATE_ORDER_KEY_IGN: word 0 of a FIRST / LAST pair, the row's order key (sd_device.h ORDER_EMPTY_FIRST) with
// its NULL flag; _IGN (ignoreNulls): the empty key for a NULL value, so the row does not count.  GATE_ORDER_VAL: word 1, the
// value (as MIN / MAX store it).  GATE_PAD: an always-zero slot that keeps the pairs at even slot indexes
enum SlotGate { GATE_VALUE = 0, GATE_NONNULL_COUNT = 1, GATE_ONE = 2, GATE_VALUE_HI32 = 3, GATE_VALUE_LO32 = 4, GATE_STRREF = 5,
                GATE_LIMB0 = 6, GATE_LIMB1 = 7, GATE_LIMB2 = 8, GATE_LIMB3 = 9, GATE_DECREF = 10,
                GATE_POW1 = 11, GATE_POW2 = 12, GATE_POW3 = 13, GATE_POW4 = 14,
                GATE_PAIR_X = 15, GATE_PAIR_Y = 16, GATE_PAIR_XY = 17, GATE_PAIR_XX = 18, GATE_PAIR_YY = 19,
                GATE_ORDER_KEY = 20, GATE_ORDER_KEY_IGN = 21, GATE_ORDER_VAL = 22, GATE_PAD = 23 };

struct SlotSpec {
  int op;     // SLOT_*
  int node;   // input expression (-1: none)
  int gate;   // SlotGate
  int table = -1;   // GATE_STRREF: index of the column's TABLE_KEYPTR table
};

// An aggregate's function family (Spark's buffers have one shape per family; MIN vs MAX, FIRST vs LAST and ignoreNulls are
// read from AggMap.fn), and how its slots carry the first buffer value:
//   HOLD_WORD    one slot word, int64 or the double's bits by buf_type
//   HOLD_HILO    DECIMAL SUM / AVG: the high and low 32-bit halves summed in value_slot / value_slot2
//   HOLD_LIMBS   wide DECIMAL SUM / AVG: four 32-bit limbs summed in limb_slot[0..3]
//   HOLD_REF     the device address of the value's [len][bytes] record (STRING, DECIMAL wider than 18 digits)
//   HOLD_SHIFTED moment / two-input sums around the group's K words
// build_slots (sd_codegen.cpp) decides both; sd_aggregate.cpp turns slots into Spark's buffers by them
enum AggFamily { AGG_COUNT = 0, AGG_SUM = 1, AGG_AVG = 2, AGG_MINMAX = 3, AGG_MOMENT = 4, AGG_PAIR = 5, AGG_ORDER = 6 };
enum AggHold { HOLD_WORD = 0, HOLD_HILO = 1, HOLD_LIMBS = 2, HOLD_REF = 3, HOLD_SHIFTED = 4 };

// how an aggregate's buffer fields map to slots
struct AggMap {
  int fn;
  int family;       // AggFamily
  int hold;         // AggHold
  int value_slot;   // SUM/AVG sum, MIN/MAX value, COUNT count
  int count_slot;   // AVG count; SUM/MIN/MAX non-null count when the buffer is nullable (-1 otherwise)
  int buf_type;     // sd_type of the (first) buffer field
  int buf_nullable;
  int value_slot2;  // HOLD_HILO: the low-half slot (value_slot holds the high half); -1 otherwise
  int in_ps;        // DECIMAL input: (precision << 8) | scale; 0 otherwise
  int buf_ps;       // DECIMAL buffer: SUM/AVG (p + 10, s) bounded to 38; MIN/MAX = input
  int limb_slot[4]; // HOLD_LIMBS: the slots of limbs 0..3 (value_slot = limb 3); else -1
  int shift;        // moment aggregate: index of its input's shift in PlanSpec.shifts (count_slot = n, value_slot = S_1); else -1
  int pow_slot[4];  // moment aggregate: S_1..S_order; else -1
  int shift_y;      // two-input aggregate: index of its y shift (`shift` is the x shift; count_slot = n, value_slot = S_xy); else -1
  int pair_slot[5]; // two-input aggregate: S_x, S_y, S_xy, S_xx, S_yy (the last two CORR only); else -1
  int order_slot;   // FIRST / LAST: the pair's key slot (value_slot = order_slot + 1 holds the value); else -1
};

// a moment aggregate's highest power: STDDEV_* / VAR_* 2, SKEWNESS 3, KURTOSIS 4
inline int moment_order(int fn) { return fn == SD_AGG_KURTOSIS ? 4 : fn == SD_AGG_SKEWNESS ? 3 : 2; }

// one shift K of a plan's moment sums (its K words are not slots, sd_device.h SHIFT_EMPTY): every moment aggregate over the
// same input shares it and its S_j slots
struct ShiftSpec {
  int order;        // highest power summed
  int pow_slot[4];  // S_1..S_order
};

// the cross term of a two-input aggregate's shifts: S_xy = sum (x - Kx)(y - Ky).  Its x and y shifts are ordinary ShiftSpecs
// (order 1, or 2 when CORR needs the squares); COVAR_* and CORR over the same PAIR share them, a moment aggregate over x does not
struct PairSpec {
  int shift_x, shift_y;
  int xy_slot;
};

// field type codes used for rows on the host: sd_type in the low byte, DECIMAL precision/scale above it
inline int field_type(int sd_type, int ps) { return sd_type == SD_DECIMAL ? (sd_type | (ps << 8)) : sd_type; }
inline int ft_base(int ft) { return ft & 0xff; }
inline int ft_precision(int ft) { return (ft >> 16) & 0xff; }
inline int ft_scale(int ft) { return (ft >> 8) & 0xff; }

struct PlanSpec {
  // deep copy of the descriptor
  std::vector<sd_column> cols;
  std::vector<sd_expr> exprs;
  std::vector<int32_t> keys;
  std::vector<sd_agg> aggs;
  std::vector<int32_t> proj;
  std::vector<int32_t> literal_types;
  int filter = -1;
  int flags = 0;                     // sd_plan_desc.flags (SD_PLAN_MUTATE)
  // grouping sets: the descriptor's last key was this SD_OP_GROUPING_ID node; `keys` are the GROUP BY expressions before it
  // (the scan kernel is the plain GROUP BY's), `sets` its masks.  -1 / empty otherwise
  int gid_node = -1;
  std::vector<uint32_t> sets;
  int out_keys() const { return (int)keys.size() + (gid_node >= 0 ? 1 : 0); }   // key fields of partial / final rows
  // analysis
  std::vector<int> expr_nullable;
  std::vector<int> kinds;            // K_* per scan column
  std::vector<char> lit_wide;        // per literal slot: 1 when it holds a wide DECIMAL (value given as bytes)
  std::vector<TableSpec> tables;
  std::vector<SlotSpec> slots;
  std::vector<AggMap> agg_map;
  std::vector<ShiftSpec> shifts;     // moment aggregates' shifts: K words [group][shift] beside the slots
  std::vector<PairSpec> pairs;       // two-input aggregates' cross terms over two of those shifts
  int norder = 0;                    // FIRST / LAST pairs (sd_device.h SLOT_FIRST)
  int rows_slot = -1;                // COUNT(*)-like slot that tells which groups exist
  int mode = 0;                      // MODE_NOKEY | MODE_GROUPS | MODE_HASH | MODE_PROJECT | MODE_MUTATE
  int rpt = 4;                       // rows per thread per tile (2, 4, 8)
  int min_ctas = 2;                  // __launch_bounds__ min CTAs per SM (= target CTAs per SM)
  int stages = 1;                    // > 0: staged fast path (producer warp + cp.async.bulk ring); 0: direct loads
  int lit_nullable = 0;              // 1: literal slots may be NULL at run time (separate kernel variant)
  int slow_paths = 0;                // 1: kernel variant that also carries the per-row decode / delta / delete paths
  int reg_groups = 0;                // > 0: MODE_GROUPS table held in registers for up to this many groups
  std::string signature;             // canonical text of everything the generated code depends on
  std::string struct_name;           // Plan_<hash of signature>
  std::string source;                // the generated PLAN struct (CUDA C++)
  std::vector<int32_t> desc_keys;    // the descriptor's keys (with the GROUPING_ID node)
  sd_plan_desc desc_view() const;    // a descriptor pointing into the vectors above
};

// kernel-shape options; -1 = heuristic default (overridable with SD_TUNE_RPT / SD_TUNE_MIN_CTAS / SD_TUNE_STAGES)
struct CodegenOptions {
  int rpt = -1;
  int min_ctas = -1;
  int stages = -1;
  int reg_groups = 0;
  int lit_nullable = 0;
  int slow_paths = 0;
  int force_hash = 0;   // keyed plans: use the hash table even when all keys are dictionary strings
};

// Analyse + generate.  Returns SD_OK or an sd_status with `err` set.
int analyze_plan(const sd_plan_desc* desc, PlanSpec& out, std::string& err, const CodegenOptions* opt = nullptr);

// Host evaluation of a string predicate node for one dictionary entry (used to fill truth tables):
// returns 0 FALSE, 1 TRUE, 2 NULL.  `s == nullptr` means the NULL code.
int eval_string_predicate(const PlanSpec& p, int node, const char* s, int slen, const sd_literal* lits);
// byte-wise comparison of two strings: < 0, 0, > 0
int cmp_bytes(const char* a, int la, const char* b, int lb);

int sum_buffer_type(int t);
// (precision << 8) | scale of a DECIMAL-typed expression node
int decimal_ps(const PlanSpec& p, int node);
bool type_is_integral(int t);
bool type_is_fp(int t);
int kind_of_type(int t);
// a DECIMAL of more than 18 digits: unscaled values do not fit int64 (records by reference in the kernel, __int128 values)
inline bool wide_decimal(int type, int precision) { return type == SD_DECIMAL && precision > 18; }
bool node_is_wide(const PlanSpec& p, int node);
// K_* of a scan column (a wide DECIMAL column travels as the 32-bit position of its record, like a raw STRING)
int kind_of_column(const sd_column& c);

}  // namespace sd
#endif
