// sd_aggregate.h -- the host side of Spark's aggregate buffers: partial / final row schemas, UnsafeRow fields, the partial
// buffers of a group from its slots, and the merge and evaluation of partial rows.  Host only: no CUDA header.
#ifndef SD_AGGREGATE_H
#define SD_AGGREGATE_H

#include <cstdint>
#include <string>
#include <unordered_map>
#include <vector>

#include "sd_codegen.h"

namespace sd {

// ---- host values (stats rows, partial rows) -------------------------------------------------------
typedef __int128 i128;
struct HVal {
  bool isnull = false;
  int64_t i = 0;
  double d = 0;
  i128 w = 0;      // DECIMAL unscaled value (any precision); `i` mirrors it when the precision is <= 18
  // merge of wide-DECIMAL SUM / AVG buffers (wide_acc_add): the exact total as acc_hi * 2^64 + acc_lo, and whether an input
  // had already overflowed
  unsigned __int128 acc_lo = 0;
  i128 acc_hi = 0;
  bool acc = false, ovf = false;
  std::string s;
};
// BigInteger(bytes): big-endian two's complement, 1..16 bytes (a wide DECIMAL record's or literal's unscaled value)
i128 dec_from_bytes(const uint8_t* b, size_t n);
int cmp_str(const std::string& a, const std::string& b);
int cmp_hval(const HVal& a, const HVal& b, int ft);

// field `idx` of a Spark UnsafeRow with `nfields` fields (SURVEY.md Appendix B.9)
bool unsafe_field(const uint8_t* row, int64_t len, int nfields, int idx, int ftype, HVal* out);
void emit_unsafe_row(std::vector<uint8_t>& out, const std::vector<int>& types, const std::vector<HVal>& vals);

// partial-row field types (keys ++ aggregate buffers) as field_type codes
std::vector<int> partial_field_types(const PlanSpec& p);

// bytes of the [len][bytes] records that HOLD_REF slots point at, by device address
typedef std::unordered_map<uint64_t, std::string> StrMap;
// partial-row fields of one group from its slot values `sv` and its moment / pair aggregates' K words `kw`
void append_agg_fields(const PlanSpec& sp, const uint64_t* sv, const uint64_t* kw, std::vector<HVal>& vals, const StrMap* strs);

// partial rows of several partitions merged by key.  evaluate = true: SnappyHashAggregateExec(Final) / CollectAggregateExec,
// merged buffers -> results (avg = sum / count); false: the merged PARTIAL rows (keys ++ buffers), what a combiner in front
// of the final stage emits.  Returns SD_OK or an sd_status with `err` set.
int merge_rows(const PlanSpec& sp, const void* partial_rows, int64_t len, bool evaluate, std::vector<uint8_t>& out,
               int64_t* out_nrows, std::string& err);

}  // namespace sd
#endif
