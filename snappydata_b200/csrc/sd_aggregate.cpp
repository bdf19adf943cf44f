// sd_aggregate.cpp -- the host side of Spark's aggregate buffers.  build_slots (sd_codegen.cpp) decides how each aggregate's
// buffers sit in slots (AggMap.family, AggMap.hold); everything here reads that decision:
//   slots -> partial buffers          SnappyHashAggregateExec partial output, SnappyHashAggregateExec.scala:1148-1178
//   merge / evaluate of partial rows  CollectAggregateExec / final merge, CollectAggregateExec.scala:67-121
#include "sd_aggregate.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>

namespace sd {

static inline int32_t rd_i32(const uint8_t* p) { int32_t v; memcpy(&v, p, 4); return v; }
static inline int16_t rd_i16(const uint8_t* p) { int16_t v; memcpy(&v, p, 2); return v; }
static inline int64_t rd_i64(const uint8_t* p) { int64_t v; memcpy(&v, p, 8); return v; }
static inline double rd_f64(const uint8_t* p) { double v; memcpy(&v, p, 8); return v; }
static inline float rd_f32(const uint8_t* p) { float v; memcpy(&v, p, 4); return v; }
static inline double u2f(uint64_t u) { double d; memcpy(&d, &u, 8); return d; }

// ---- host values and UnsafeRows -----------------------------------------------------------------------
static i128 pow10_128(int k) { i128 r = 1; for (int j = 0; j < k; j++) r *= 10; return r; }
i128 dec_from_bytes(const uint8_t* b, size_t n) {
  unsigned __int128 u = (unsigned __int128)(i128)(int8_t)b[0];
  for (size_t k = 1; k < n; k++) u = (u << 8) | b[k];
  return (i128)u;
}

int cmp_str(const std::string& a, const std::string& b) { return cmp_bytes(a.data(), (int)a.size(), b.data(), (int)b.size()); }
static int cmp_f64(double x, double y) {   // Utils.nanSafeCompareDoubles
  const bool xn = std::isnan(x), yn = std::isnan(y);
  if (xn || yn) return xn && yn ? 0 : (xn ? 1 : -1);
  return x < y ? -1 : (x > y ? 1 : 0);
}
int cmp_hval(const HVal& a, const HVal& b, int ft) {
  const int t = ft_base(ft);
  if (t == SD_STRING) return cmp_str(a.s, b.s);
  if (type_is_fp(t)) return cmp_f64(a.d, b.d);
  if (t == SD_DECIMAL) return a.w < b.w ? -1 : (a.w > b.w ? 1 : 0);
  return a.i < b.i ? -1 : (a.i > b.i ? 1 : 0);
}

bool unsafe_field(const uint8_t* row, int64_t len, int nfields, int idx, int ftype, HVal* out) {
  const int64_t bits = ((nfields + 63) / 64) * 8;
  if (idx < 0 || idx >= nfields || bits + 8 * (int64_t)nfields > len) return false;
  *out = HVal();
  if (row[idx >> 3] & (1u << (idx & 7))) { out->isnull = true; return true; }
  const uint8_t* slot = row + bits + 8 * (int64_t)idx;
  const int type = ft_base(ftype);
  const int64_t ol = rd_i64(slot), off = ol >> 32, ln = ol & 0xffffffff;   // a variable-length field's offset and size
  if (type == SD_DECIMAL) {   // UnsafeRow.getDecimal: long for precision <= 18, else BigInteger bytes (big-endian two's complement)
    if (ft_precision(ftype) <= 18) { out->i = ol; out->w = out->i; return true; }
    if (off < 0 || ln > 16 || off + ln > len) return false;
    out->w = ln > 0 ? dec_from_bytes(row + off, (size_t)ln) : 0;
    out->i = (int64_t)out->w;
    return true;
  }
  switch (type) {
    case SD_STRING:
      if (off < 0 || off + ln > len) return false;
      out->s.assign(reinterpret_cast<const char*>(row + off), (size_t)ln);
      break;
    case SD_BOOLEAN: out->i = slot[0] != 0; break;
    case SD_BYTE: out->i = (int8_t)slot[0]; break;
    case SD_SHORT: out->i = rd_i16(slot); break;
    case SD_INT: case SD_DATE: out->i = rd_i32(slot); break;
    case SD_FLOAT: out->d = rd_f32(slot); break;
    case SD_DOUBLE: out->d = rd_f64(slot); break;
    default: out->i = ol; break;
  }
  return true;
}

void emit_unsafe_row(std::vector<uint8_t>& out, const std::vector<int>& types, const std::vector<HVal>& vals) {
  const int n = (int)types.size();
  const int64_t bits = ((n + 63) / 64) * 8, fixed = bits + 8 * (int64_t)n;
  int64_t var = 0;
  for (int i = 0; i < n; i++) {
    if (types[i] == SD_STRING && !vals[i].isnull) var += ((int64_t)vals[i].s.size() + 7) & ~int64_t(7);
    if (ft_base(types[i]) == SD_DECIMAL && ft_precision(types[i]) > 18) var += 16;   // always reserved (UnsafeRowWriter.write(Decimal))
  }
  const int64_t sz = fixed + var;
  const size_t base = out.size();
  out.resize(base + 8 + sz, 0);
  uint8_t* r = out.data() + base;
  memcpy(r, &sz, 8);
  r += 8;
  int64_t voff = fixed;
  for (int i = 0; i < n; i++) {
    uint8_t* slot = r + bits + 8 * (int64_t)i;
    if (ft_base(types[i]) == SD_DECIMAL) {
      const bool wide = ft_precision(types[i]) > 18;
      if (vals[i].isnull) {
        r[i >> 3] |= (uint8_t)(1u << (i & 7));
        if (wide) { const int64_t ol = voff << 32; memcpy(slot, &ol, 8); voff += 16; }   // offset kept, size 0
        continue;
      }
      if (!wide) { const int64_t v = (int64_t)vals[i].w; memcpy(slot, &v, 8); continue; }
      // BigInteger.toByteArray(): minimal big-endian two's complement
      uint8_t be[16];
      i128 v = vals[i].w;
      for (int k = 15; k >= 0; k--) { be[k] = (uint8_t)(v & 0xff); v >>= 8; }
      int first = 0;
      while (first < 15 && ((be[first] == 0x00 && !(be[first + 1] & 0x80)) || (be[first] == 0xff && (be[first + 1] & 0x80)))) first++;
      const int nb = 16 - first;
      memcpy(r + voff, be + first, (size_t)nb);
      const int64_t ol = (voff << 32) | (int64_t)nb;
      memcpy(slot, &ol, 8);
      voff += 16;
      continue;
    }
    if (vals[i].isnull) { r[i >> 3] |= (uint8_t)(1u << (i & 7)); continue; }
    switch (types[i]) {
      case SD_STRING: {
        const int64_t ol = (voff << 32) | (uint32_t)vals[i].s.size();
        memcpy(slot, &ol, 8);
        memcpy(r + voff, vals[i].s.data(), vals[i].s.size());
        voff += ((int64_t)vals[i].s.size() + 7) & ~int64_t(7);
        break;
      }
      case SD_BOOLEAN: slot[0] = vals[i].i != 0; break;
      case SD_BYTE: { int8_t v = (int8_t)vals[i].i; memcpy(slot, &v, 1); break; }
      case SD_SHORT: { int16_t v = (int16_t)vals[i].i; memcpy(slot, &v, 2); break; }
      case SD_INT: case SD_DATE: { int32_t v = (int32_t)vals[i].i; memcpy(slot, &v, 4); break; }
      case SD_FLOAT: { float v = (float)vals[i].d; memcpy(slot, &v, 4); break; }
      case SD_DOUBLE: memcpy(slot, &vals[i].d, 8); break;
      default: memcpy(slot, &vals[i].i, 8); break;
    }
  }
}

// ---- buffer layout ----------------------------------------------------------------------------------
// partial-row buffer fields of an aggregate: AVG [sum, count]; moments [n, avg, m2, (m3, (m4))]; COVAR_* [n, xAvg, yAvg, ck];
// CORR [n, xAvg, yAvg, ck, xMk, yMk]; FIRST / LAST [value, valueSet]; others one
static int buffer_fields(const AggMap& m) {
  switch (m.family) {
    case AGG_AVG: case AGG_ORDER: return 2;
    case AGG_MOMENT: return 1 + moment_order(m.fn);
    case AGG_PAIR: return m.fn == SD_AGG_CORR ? 6 : 4;
    default: return 1;
  }
}

static void key_field_types(const PlanSpec& p, std::vector<int>& t) {
  for (int k : p.keys) t.push_back(field_type(p.exprs[k].type, p.exprs[k].type == SD_DECIMAL ? decimal_ps(p, k) : 0));
  if (p.gid_node >= 0) t.push_back(SD_INT);   // spark_grouping_id
}
std::vector<int> partial_field_types(const PlanSpec& p) {
  std::vector<int> t;
  key_field_types(p, t);
  for (auto& m : p.agg_map) {   // the first field has the buffer type; AVG's count is a LONG, FIRST / LAST's valueSet a BOOLEAN
    t.push_back(field_type(m.buf_type, m.buf_ps));
    t.insert(t.end(), (size_t)buffer_fields(m) - 1, m.family == AGG_AVG ? SD_LONG : m.family == AGG_ORDER ? SD_BOOLEAN : SD_DOUBLE);
  }
  return t;
}
// final-row field types: keys ++ results
static std::vector<int> final_field_types(const PlanSpec& p) {
  std::vector<int> t;
  key_field_types(p, t);
  for (auto& m : p.agg_map) {
    if (m.family == AGG_AVG) {
      if (m.buf_type == SD_DECIMAL) {   // Average.resultType: DecimalType.bounded(p + 4, s + 4)
        const int pr = std::min(38, (m.in_ps >> 8) + 4), sc = std::min(38, (m.in_ps & 0xff) + 4);
        t.push_back(field_type(SD_DECIMAL, (pr << 8) | sc));
      } else t.push_back(SD_DOUBLE);
    } else t.push_back(field_type(m.buf_type, m.buf_ps));
  }
  return t;
}

// ---- wide-DECIMAL sums (HOLD_LIMBS) -------------------------------------------------------------------
// SUM / AVG buffers of a wide DECIMAL: a total of more than min(38, p + 10) digits is carried through partial rows (and every
// merge of them) as pow10_128(precision), a value no in-range total reaches, so the final result is NULL however the rows
// were split into partitions -- the rule one execution applies to all its rows
static bool wide_sum_overflowed(i128 v, int prec) { return v >= pow10_128(prec) || v <= -pow10_128(prec); }
// merges add partial totals exactly (each in-range one is below 2^127, so 64-bit halves summed in 128 bits cannot wrap);
// the total is NULL when an input had overflowed or the exact sum of all of them needs more than `prec` digits
static void wide_acc_add(HVal& b, const HVal& in, int prec) {
  if (!b.acc) {
    b.acc = true;
    b.ovf = wide_sum_overflowed(b.w, prec);
    b.acc_lo = (uint64_t)b.w;
    b.acc_hi = b.w >> 64;
  }
  b.ovf = b.ovf || wide_sum_overflowed(in.w, prec);
  b.acc_lo += (uint64_t)in.w;
  b.acc_hi += in.w >> 64;
}
static void wide_acc_finish(HVal& b, int prec) {
  if (!b.acc) return;
  const i128 hi = b.acc_hi + (i128)(b.acc_lo >> 64);
  const uint64_t lo = (uint64_t)b.acc_lo;
  b.acc = false;
  if (b.ovf || hi < -((i128)1 << 63) || hi >= ((i128)1 << 63)) b.w = pow10_128(prec);
  else {
    b.w = (i128)(((unsigned __int128)hi << 64) | lo);
    if (wide_sum_overflowed(b.w, prec)) b.w = pow10_128(prec);
  }
  b.i = (int64_t)b.w;
}

// l3 * 2^96 + l2 * 2^64 + l1 * 2^32 + l0 (l0..l2: sums of unsigned 32-bit limbs, l3: sum of the signed top limbs); *fits = false
// when the total is outside the int128 range
static i128 limbs_to_i128(uint64_t l0, uint64_t l1, uint64_t l2, int64_t l3, bool* fits) {
  uint64_t c = l0;
  const uint64_t d0 = c & 0xffffffffull;
  c = l1 + (c >> 32);
  const uint64_t d1 = c & 0xffffffffull;
  c = l2 + (c >> 32);
  const uint64_t d2 = c & 0xffffffffull;
  const i128 top = (i128)l3 + (i128)(c >> 32);
  *fits = top >= -((i128)1 << 31) && top < ((i128)1 << 31);
  if (!*fits) return 0;
  const unsigned __int128 low = ((unsigned __int128)d2 << 64) | ((unsigned __int128)d1 << 32) | d0;
  return (i128)(((unsigned __int128)top << 96) | low);
}

// ---- slots -> buffers: the value ----------------------------------------------------------------------
// the first buffer value of a group from its slot word(s), as AggMap.hold says they carry it
static HVal decode_value(const AggMap& m, const uint64_t* sv, const StrMap* strs) {
  HVal v;
  const uint64_t raw = sv[m.value_slot];
  switch (m.hold) {
    case HOLD_HILO:   // high and low halves summed separately
      v.w = (i128)(int64_t)sv[m.value_slot] * ((i128)1 << 32) + (i128)(int64_t)sv[m.value_slot2];
      break;
    case HOLD_LIMBS: {   // four 32-bit limbs summed separately; an overflowed total is sticky (wide_acc_add)
      bool fits = false;
      v.w = limbs_to_i128(sv[m.limb_slot[0]], sv[m.limb_slot[1]], sv[m.limb_slot[2]], (int64_t)sv[m.limb_slot[3]], &fits);
      if (!fits || wide_sum_overflowed(v.w, m.buf_ps >> 8)) v.w = pow10_128(m.buf_ps >> 8);
      break;
    }
    case HOLD_REF: {   // the device address of a [len][bytes] record, 0 = none
      const StrMap::const_iterator it = strs ? strs->find(raw) : StrMap::const_iterator();
      if (raw == 0 || !strs || it == strs->end()) v.isnull = true;
      else if (m.buf_type == SD_STRING) { v.s = it->second; return v; }
      else if (it->second.empty() || it->second.size() > 16) v.isnull = true;
      else v.w = dec_from_bytes(reinterpret_cast<const uint8_t*>(it->second.data()), it->second.size());
      break;
    }
    default:   // HOLD_WORD
      if (type_is_fp(m.buf_type)) { memcpy(&v.d, &raw, 8); return v; }
      v.w = (int64_t)raw;
      break;
  }
  v.i = (int64_t)v.w;
  return v;
}

// ---- AVG ------------------------------------------------------------------------------------------------
// Average.evaluateExpression: sum / count, NULL when count == 0; `ft` is the result's field type.  DECIMAL: Cast(Cast(sum,
// DECIMAL(p+14,s+4)) / Cast(count, ...), DECIMAL(p+4,s+4)), the quotient at scale s+4, HALF_UP.  sum * 10^k may not fit 128
// bits for a wide input: q0 = sum / count, then the k more digits from the remainder (|remainder| * 10^k < 2^63 * 10^4); a
// q0 of more than precision - k digits cannot fit
static HVal avg_result(const AggMap& m, const HVal* b, int ft) {
  HVal v;
  const int64_t cnt = b[1].i;
  if (cnt == 0) v.isnull = true;
  else if (m.buf_type != SD_DECIMAL) v.d = b[0].d / (double)cnt;
  else {
    const int kk = ft_scale(ft) - (m.in_ps & 0xff), pr = ft_precision(ft);
    const i128 sum = b[0].w, den = cnt, q0 = sum / den, r0 = sum % den;
    // a wide sum of more than p + 10 digits is NULL: so is the average
    if ((m.hold == HOLD_LIMBS && wide_sum_overflowed(sum, m.buf_ps >> 8)) || q0 >= pow10_128(pr - kk) || q0 <= -pow10_128(pr - kk)) v.isnull = true;
    else {
      const i128 num1 = r0 * pow10_128(kk);
      i128 q = q0 * pow10_128(kk) + num1 / den, rem = num1 % den;
      if (rem < 0) rem = -rem;
      if (2 * rem >= den) q += (sum < 0 ? -1 : 1);
      if (q >= pow10_128(pr) || q <= -pow10_128(pr)) v.isnull = true;
      else { v.w = q; v.i = (int64_t)q; }
    }
  }
  return v;
}

// ---- STDDEV / VARIANCE / SKEWNESS / KURTOSIS ------------------------------------------------------------
// Spark's buffers [n, avg, m2, (m3, (m4))] from n and S_j = sum (x - K)^j
static void moment_buffers(const AggMap& m, const uint64_t* sv, const uint64_t* kw, int64_t cnt, HVal* b) {
  if (cnt <= 0) return;
  const int order = moment_order(m.fn);
  const double n = (double)cnt, K = u2f(kw[m.shift]), S1 = u2f(sv[m.pow_slot[0]]), S2 = u2f(sv[m.pow_slot[1]]);
  const double S3 = order >= 3 ? u2f(sv[m.pow_slot[2]]) : 0.0, S4 = order >= 4 ? u2f(sv[m.pow_slot[3]]) : 0.0;
  const double d = S1 / n;
  b[0].d = n;
  b[1].d = K + d;
  const double m2 = S2 - n * d * d;
  b[2].d = m2 < 0 ? 0.0 : m2;   // rounding; a NaN stays NaN
  if (order >= 3) b[3].d = S3 - 3 * d * S2 + 2 * n * d * d * d;
  if (order >= 4) b[4].d = S4 - 4 * d * S3 + 6 * d * d * S2 - 3 * n * d * d * d * d;
}
// CentralMomentAgg (Spark 2.1.1) on the buffers b[0..order] = [n, avg, m2, (m3, (m4))]: mergeExpressions ...
static void moment_merge(HVal* b, const HVal* in, int order) {
  const double n1 = b[0].d, n2 = in[0].d, n = n1 + n2;
  const double delta = in[1].d - b[1].d, dN = n == 0.0 ? 0.0 : delta / n;
  const double m2a = b[2].d, m2b = in[2].d;
  const double m3a = order >= 3 ? b[3].d : 0.0, m3b = order >= 3 ? in[3].d : 0.0;
  b[0].d = n;
  b[1].d = b[1].d + dN * n2;
  b[2].d = m2a + m2b + delta * dN * n1 * n2;
  if (order >= 3) b[3].d = m3a + m3b + dN * dN * delta * n1 * n2 * (n1 - n2) + 3.0 * dN * (n1 * m2b - n2 * m2a);
  if (order >= 4)
    b[4].d = b[4].d + in[4].d + dN * dN * dN * delta * n1 * n2 * (n1 * n1 - n1 * n2 + n2 * n2) + 6.0 * dN * dN * (n1 * n1 * m2b + n2 * n2 * m2a) +
             4.0 * dN * (n1 * m3b - n2 * m3a);
}
// ... and evaluateExpression: NULL without input; stddev / variance are the SAMP forms
static HVal moment_result(int fn, const HVal* b) {
  HVal v;
  const double n = b[0].d, m2 = b[2].d;
  if (n == 0.0) { v.isnull = true; return v; }
  switch (fn) {
    case SD_AGG_VAR_POP: v.d = m2 / n; break;
    case SD_AGG_STDDEV_POP: v.d = std::sqrt(m2 / n); break;
    case SD_AGG_VAR_SAMP: v.d = n == 1.0 ? NAN : m2 / (n - 1.0); break;
    case SD_AGG_STDDEV_SAMP: v.d = n == 1.0 ? NAN : std::sqrt(m2 / (n - 1.0)); break;
    case SD_AGG_SKEWNESS: v.d = m2 == 0.0 ? NAN : std::sqrt(n) * b[3].d / std::sqrt(m2 * m2 * m2); break;
    default: v.d = m2 == 0.0 ? NAN : n * b[4].d / (m2 * m2) - 3.0; break;   // SD_AGG_KURTOSIS
  }
  return v;
}

// ---- COVAR_POP / COVAR_SAMP / CORR ----------------------------------------------------------------------
// Spark's buffers [n, xAvg, yAvg, ck, (xMk, yMk)] from n, S_x, S_y, S_xy (, S_xx, S_yy)
static void pair_buffers(const AggMap& m, const uint64_t* sv, const uint64_t* kw, int64_t cnt, HVal* b) {
  if (cnt <= 0) return;
  const double n = (double)cnt, Kx = u2f(kw[m.shift]), Ky = u2f(kw[m.shift_y]);
  const double Sx = u2f(sv[m.pair_slot[0]]), Sy = u2f(sv[m.pair_slot[1]]), Sxy = u2f(sv[m.pair_slot[2]]);
  const double dx = Sx / n, dy = Sy / n;
  const int nb = m.fn == SD_AGG_CORR ? 6 : 4;
  b[0].d = n;
  if (!std::isfinite(Kx) || !std::isfinite(Ky) || !std::isfinite(Sx) || !std::isfinite(Sy)) {
    // a counted row had a NaN or +-Inf x or y (its shifted value, or the group's K, is not finite): NaN, not the +-Inf
    // some shifted sums would give
    for (int j = 1; j < nb; j++) b[j].d = NAN;
    return;
  }
  b[1].d = Kx + dx;
  b[2].d = Ky + dy;
  b[3].d = Sxy - n * dx * dy;
  if (nb == 6) {   // >= 0 despite rounding (S_x, S_y are finite here)
    b[4].d = std::max(0.0, u2f(sv[m.pair_slot[3]]) - n * dx * dx);
    b[5].d = std::max(0.0, u2f(sv[m.pair_slot[4]]) - n * dy * dy);
  }
}
// Covariance / Corr (Spark 2.1.1) on the buffers [n, xAvg, yAvg, ck, (xMk, yMk)]: mergeExpressions ...
static void pair_merge(HVal* b, const HVal* in, bool corr) {
  const double n1 = b[0].d, n2 = in[0].d, n = n1 + n2;
  const double dx = in[1].d - b[1].d, dxN = n == 0.0 ? 0.0 : dx / n;
  const double dy = in[2].d - b[2].d, dyN = n == 0.0 ? 0.0 : dy / n;
  b[0].d = n;
  b[1].d = b[1].d + dxN * n2;
  b[2].d = b[2].d + dyN * n2;
  b[3].d = b[3].d + in[3].d + dx * dyN * n1 * n2;
  if (corr) {
    b[4].d = b[4].d + in[4].d + dx * dxN * n1 * n2;
    b[5].d = b[5].d + in[5].d + dy * dyN * n1 * n2;
  }
}
// ... and evaluateExpression: NULL without input
static HVal pair_result(int fn, const HVal* b) {
  HVal v;
  const double n = b[0].d, ck = b[3].d;
  if (n == 0.0) { v.isnull = true; return v; }
  switch (fn) {
    case SD_AGG_COVAR_POP: v.d = ck / n; break;
    case SD_AGG_COVAR_SAMP: v.d = n == 1.0 ? NAN : ck / (n - 1.0); break;
    default: v.d = n == 1.0 ? NAN : ck / std::sqrt(b[4].d * b[5].d); break;   // SD_AGG_CORR
  }
  return v;
}

// ---- the stages of one aggregate: its buffers b[0 .. buffer_fields(m)) ------------------------------------
// of one group, from its slots
static void from_slots(const PlanSpec& sp, const AggMap& m, const uint64_t* sv, const uint64_t* kw, const StrMap* strs, HVal* b) {
  const int64_t cnt = m.count_slot >= 0 ? (int64_t)sv[m.count_slot] : 1;
  switch (m.family) {
    case AGG_MOMENT: moment_buffers(m, sv, kw, cnt, b); return;
    case AGG_PAIR: pair_buffers(m, sv, kw, cnt, b); return;
    case AGG_ORDER: {   // [value, valueSet] from the pair (order key, value)
      const uint64_t key = sv[m.order_slot];
      b[1].i = key != slot_initial(sp.slots[(size_t)m.order_slot].op);
      if (!b[1].i || (key & 1ull)) b[0].isnull = true;   // no row, or the row's value is NULL
      else b[0] = decode_value(m, sv, strs);
      return;
    }
    case AGG_AVG: b[1].i = cnt; break;
    default: break;
  }
  b[0] = decode_value(m, sv, strs);
  if (m.buf_nullable && cnt == 0) b[0].isnull = true;   // SUM / MIN / MAX without a non-null input
}
// mergeExpressions: `in` into `b`
static void merge_buffers(const PlanSpec& sp, const AggMap& m, HVal* b, const HVal* in) {
  const int prec = m.buf_ps >> 8;
  switch (m.family) {
    case AGG_COUNT: b[0].i += in[0].i; break;
    case AGG_SUM:   // NULL + NULL = NULL, otherwise NULLs count as 0
      if (in[0].isnull) break;
      if (m.hold == HOLD_LIMBS) { if (b[0].isnull) b[0].w = in[0].w; else wide_acc_add(b[0], in[0], prec); }
      else if (m.hold == HOLD_HILO) { b[0].w = (b[0].isnull ? (i128)0 : b[0].w) + in[0].w; b[0].i = (int64_t)b[0].w; }
      else if (m.buf_type == SD_DOUBLE) b[0].d = (b[0].isnull ? 0.0 : b[0].d) + in[0].d;
      else b[0].i = (int64_t)((uint64_t)(b[0].isnull ? 0 : b[0].i) + (uint64_t)in[0].i);
      b[0].isnull = false;
      break;
    case AGG_AVG:   // [sum, count]
      if (m.hold == HOLD_LIMBS) wide_acc_add(b[0], in[0], prec);
      else if (m.hold == HOLD_HILO) { b[0].w += in[0].w; b[0].i = (int64_t)b[0].w; }
      else b[0].d += in[0].d;
      b[1].i += in[1].i;
      break;
    case AGG_MINMAX:
      if (in[0].isnull) break;
      if (b[0].isnull) { b[0] = in[0]; break; }
      if (const int c = cmp_hval(in[0], b[0], m.buf_type); (m.fn == SD_AGG_MIN && c < 0) || (m.fn == SD_AGG_MAX && c > 0)) b[0] = in[0];
      break;
    case AGG_MOMENT: moment_merge(b, in, moment_order(m.fn)); break;
    case AGG_PAIR: pair_merge(b, in, m.fn == SD_AGG_CORR); break;
    case AGG_ORDER:   // First: valueSet.left ? left : right; Last: valueSet.right ? right : left; valueSet = left || right
      if (sp.slots[(size_t)m.order_slot].op == SLOT_LAST ? in[1].i != 0 : b[1].i == 0) { b[0] = in[0]; b[1].i = b[1].i || in[1].i; }
      break;
  }
}
// evaluateExpression; `ft` is the result's field type
static HVal result_of(const AggMap& m, const HVal* b, int ft) {
  HVal v = b[0];
  switch (m.family) {
    case AGG_SUM:   // a DECIMAL sum that needs more than p+10 digits is NULL (changePrecision fails)
      if (m.buf_type == SD_DECIMAL && !v.isnull && wide_sum_overflowed(v.w, m.buf_ps >> 8)) v.isnull = true;
      return v;
    case AGG_AVG: return avg_result(m, b, ft);
    case AGG_MOMENT: return moment_result(m.fn, b);
    case AGG_PAIR: return pair_result(m.fn, b);
    default: return v;   // COUNT, MIN / MAX, and First / Last: the value
  }
}

void append_agg_fields(const PlanSpec& sp, const uint64_t* sv, const uint64_t* kw, std::vector<HVal>& vals, const StrMap* strs) {
  for (auto& m : sp.agg_map) {
    const size_t k = vals.size();
    vals.resize(k + (size_t)buffer_fields(m));
    from_slots(sp, m, sv, kw, strs, &vals[k]);
  }
}

// ---- merge of partial rows (a handful of rows per partition) ------------------------------------------------
int merge_rows(const PlanSpec& sp, const void* partial_rows, int64_t len, bool evaluate, std::vector<uint8_t>& out,
               int64_t* out_nrows, std::string& err) {
  out.clear();
  if (sp.mode == MODE_PROJECT) {   // projected rows of several partitions: concatenation
    const uint8_t* r = reinterpret_cast<const uint8_t*>(partial_rows);
    int64_t pos = 0, n = 0;
    while (pos + 8 <= len) {
      const int64_t sz = rd_i64(r + pos);
      if (sz < 0 || pos + 8 + sz > len) { err = "merge: bad row size"; return SD_ERR_INVALID; }
      pos += 8 + sz; n++;
    }
    out.assign(r, r + pos);
    if (out_nrows) *out_nrows = n;
    return 0;
  }
  const int nk = sp.out_keys();
  const std::vector<int> types = partial_field_types(sp);
  const int n = (int)types.size();
  std::vector<size_t> first;   // per aggregate: its first buffer field among a group's buffers
  for (size_t a = 0, k = 0; a < sp.agg_map.size(); k += (size_t)buffer_fields(sp.agg_map[a]), a++) first.push_back(k);
  struct Group { std::vector<HVal> keys; std::vector<HVal> bufs; };
  std::vector<Group> groups;   // insertion order
  std::map<std::string, size_t> index;
  const uint8_t* r = reinterpret_cast<const uint8_t*>(partial_rows);
  int64_t pos = 0;
  std::vector<HVal> f((size_t)n);
  std::string key;
  while (pos + 8 <= len) {
    const int64_t sz = rd_i64(r + pos);
    if (sz < 0 || pos + 8 + sz > len) { err = "sd_final_merge: bad row size"; return SD_ERR_INVALID; }
    for (int i = 0; i < n; i++)
      if (!unsafe_field(r + pos + 8, sz, n, i, types[i], &f[i])) { err = "sd_final_merge: malformed partial row"; return SD_ERR_INVALID; }
    key.clear();
    for (int k = 0; k < nk; k++) {
      key.push_back(f[k].isnull ? 'N' : 'V');
      if (!f[k].isnull) {
        if (types[k] == SD_STRING) { uint32_t l = (uint32_t)f[k].s.size(); key.append(reinterpret_cast<char*>(&l), 4); key.append(f[k].s); }
        else if (type_is_fp(types[k])) { double d = f[k].d; if (d == 0.0) d = 0.0; if (std::isnan(d)) d = NAN; key.append(reinterpret_cast<char*>(&d), 8); }
        else if (ft_base(types[k]) == SD_DECIMAL && ft_precision(types[k]) > 18) key.append(reinterpret_cast<const char*>(&f[k].w), 16);
        else key.append(reinterpret_cast<const char*>(&f[k].i), 8);
      }
    }
    auto it = nk > 0 ? index.find(key) : (groups.empty() ? index.end() : index.begin());
    if (it == index.end()) {
      index.emplace(key, groups.size());
      groups.push_back(Group());
      groups.back().keys.assign(f.begin(), f.begin() + nk);
      groups.back().bufs.assign(f.begin() + nk, f.end());
    } else {
      Group& g = groups[it->second];
      for (size_t a = 0; a < sp.agg_map.size(); a++) merge_buffers(sp, sp.agg_map[a], &g.bufs[first[a]], &f[(size_t)nk + first[a]]);
    }
    pos += 8 + sz;
  }
  if (nk == 0 && groups.empty()) {   // no-key aggregate over no partitions: one row of empty buffers
    groups.push_back(Group());
    groups.back().bufs.resize((size_t)(n - nk));
    for (size_t a = 0; a < sp.agg_map.size(); a++) {   // SUM / MIN / MAX NULL, FIRST / LAST [NULL, false], everything else 0
      const int f = sp.agg_map[a].family;
      groups.back().bufs[first[a]].isnull = f == AGG_SUM || f == AGG_MINMAX || f == AGG_ORDER;
    }
  }
  const std::vector<int> otypes = evaluate ? final_field_types(sp) : types;
  std::vector<HVal> vals;
  for (auto& g : groups) {
    for (size_t a = 0; a < sp.agg_map.size(); a++)   // a wide sum's exact total back into its value
      if (sp.agg_map[a].hold == HOLD_LIMBS) wide_acc_finish(g.bufs[first[a]], sp.agg_map[a].buf_ps >> 8);
    vals.assign(g.keys.begin(), g.keys.end());
    if (!evaluate) vals.insert(vals.end(), g.bufs.begin(), g.bufs.end());
    else
      for (size_t a = 0; a < sp.agg_map.size(); a++) vals.push_back(result_of(sp.agg_map[a], &g.bufs[first[a]], otypes[vals.size()]));
    emit_unsafe_row(out, otypes, vals);
  }
  if (out_nrows) *out_nrows = (int64_t)groups.size();
  return 0;
}

}  // namespace sd
