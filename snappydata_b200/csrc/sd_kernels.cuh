// sd_kernels.cuh -- the fused scan -> decode -> filter -> partial-aggregate kernel for sm_90a.
//
// One kernel template, specialised per plan by a small generated struct (PLAN) that supplies the
// plan's column kinds and three inline functions: filter(), group() and slots() -- the CUDA
// counterpart of the reference's WholeStageCodegen class for
//   ColumnTableScan.doProduce            core/execution/columnar/ColumnTableScan.scala:186-672
//   FilterExec.doConsume                 (Spark 2.1.1)
//   SnappyHashAggregateExec.doConsume    core/execution/aggregate/SnappyHashAggregateExec.scala:252-263
// Everything else here is hand-written: batch/tile scheduling, the per-encoding decoders
// (Uncompressed / Dictionary / BigDictionary / BooleanBitSet / RunLength, nullable or not), the
// update-delta overlay and delete mask, and the aggregation machinery.
//
// Roofline: the kernel is HBM-read bound (<= ~3 flops per loaded byte; no dense contraction, so
// tensor cores do not apply).  Design for that bound:
//   * every column read of the common case (NOT NULL or no nulls in the batch, Uncompressed or
//     int16/int32 dictionary indexes, no deltas) is ONE fully coalesced, 16-byte-aligned,
//     cache-streaming vector load per row pair per lane (16/8/4/2 bytes per lane);
//   * all loads of a tile (every column, RPT rows) are issued before the first use, so each thread
//     keeps NC * RPT/2 independent requests in flight;
//   * a persistent grid of num_SMs * CTAS_PER_SM CTAs walks (batch, chunk) work items round-robin -- no
//     per-batch launch, deterministic reduction order;
//   * aggregation never touches global atomics on the hot path: registers (no keys) or per-thread
//     private shared-memory tables laid out bank-conflict free (small group counts), reduced once per
//     CTA, then by the last CTA in fixed order.
//
// Self-contained: includes only sd_device.h so NVRTC can compile it from an in-memory string.
// Included by more than one translation unit (the plan kernels, sd_compact.cu): out-of-line helpers that are not templates
// have internal linkage.
#ifndef SD_KERNELS_CUH
#define SD_KERNELS_CUH

#include "sd_device.h"

namespace sd {

// ---- kind -> register type --------------------------------------------------------------------
template <int K> struct KindT;
template <> struct KindT<K_I8> { typedef int8_t T; };
template <> struct KindT<K_I16> { typedef int16_t T; };
template <> struct KindT<K_I32> { typedef int32_t T; };
template <> struct KindT<K_I64> { typedef int64_t T; };
template <> struct KindT<K_F32> { typedef float T; };
template <> struct KindT<K_F64> { typedef double T; };
template <> struct KindT<K_BOOL> { typedef uint8_t T; };
template <> struct KindT<K_CODE> { typedef int32_t T; };

template <int... Is> struct Seq {};
template <int N, int... Is> struct MakeSeq : MakeSeq<N - 1, N - 1, Is...> {};
template <int... Is> struct MakeSeq<0, Is...> { typedef Seq<Is...> type; };

// ---- NaN-safe total order of Spark's double/float comparisons (Utils.nanSafeCompareDoubles:
//      NaN == NaN, NaN greater than everything, -0.0 == 0.0; SURVEY.md Appendix B.5) ------------
template <class F> __device__ __forceinline__ bool f_ge(F a, F b) { return (a >= b) || (a != a); }
template <class F> __device__ __forceinline__ bool f_gt(F a, F b) { return (a > b) || ((a != a) && (b == b)); }
template <class F> __device__ __forceinline__ bool f_le(F a, F b) { return f_ge(b, a); }
template <class F> __device__ __forceinline__ bool f_lt(F a, F b) { return f_gt(b, a); }
template <class F> __device__ __forceinline__ bool f_eq(F a, F b) { return (a == b) || ((a != a) && (b != b)); }

// Java (int)/(long) casts of floating point: NaN -> 0, saturating
__device__ __forceinline__ int64_t f64_to_i64(double d) { return (d != d) ? 0 : __double2ll_rz(d); }
__device__ __forceinline__ int32_t f64_to_i32(double d) { return (d != d) ? 0 : __double2int_rz(d); }

// three-valued logic helpers for generated predicates: 0 FALSE, 1 TRUE, 2 NULL
__device__ __forceinline__ int tv_and(int a, int b) { return (a == 0 || b == 0) ? 0 : ((a == 2 || b == 2) ? 2 : 1); }
__device__ __forceinline__ int tv_or(int a, int b) { return (a == 1 || b == 1) ? 1 : ((a == 2 || b == 2) ? 2 : 0); }
__device__ __forceinline__ int tv_not(int a) { return a == 2 ? 2 : 1 - a; }

// ---- variable-width strings by their bytes: records are [len:int32 LE][bytes], unaligned (enc/Uncompressed.scala:116-161;
//      the same layout as a string dictionary entry, enc/DictionaryEncoding.scala:452-518).  Strings compare as unsigned
//      bytes, shorter first on a common prefix (UTF8String.compareTo; SURVEY.md Appendix B.5) -----------------------------
__device__ __forceinline__ int rec_len(const uint8_t* rec) {
  return (int)((uint32_t)rec[0] | ((uint32_t)rec[1] << 8) | ((uint32_t)rec[2] << 16) | ((uint32_t)rec[3] << 24));
}
static __device__ __noinline__ int str_cmp_rec(const uint8_t* rec, const uint8_t* lit, int llen) {
  const int n = rec_len(rec);
  const uint8_t* s = rec + 4;
  const int m = n < llen ? n : llen;
  for (int i = 0; i < m; i++) { const int d = (int)s[i] - (int)lit[i]; if (d) return d; }
  return n - llen;
}
static __device__ __noinline__ bool str_starts_rec(const uint8_t* rec, const uint8_t* lit, int llen) {
  if (rec_len(rec) < llen) return false;
  const uint8_t* s = rec + 4;
  for (int i = 0; i < llen; i++) if (s[i] != lit[i]) return false;
  return true;
}
static __device__ __noinline__ bool str_eq_recs(const uint8_t* a, const uint8_t* b) {
  if (a == b) return true;
  const int n = rec_len(a);
  if (n != rec_len(b)) return false;
  for (int i = 0; i < n; i++) if (a[4 + i] != b[4 + i]) return false;
  return true;
}
static __device__ __noinline__ int str_cmp_recs(const uint8_t* a, const uint8_t* b) {   // UTF8String.compareTo on two records
  const int na = rec_len(a), nb = rec_len(b), m = na < nb ? na : nb;
  for (int i = 0; i < m; i++) { const int d = (int)a[4 + i] - (int)b[4 + i]; if (d) return d; }
  return na - nb;
}
static __device__ __noinline__ uint64_t str_hash_rec(const uint8_t* rec) {   // FNV-1a over the bytes
  const int n = rec_len(rec);
  uint64_t h = 1469598103934665603ull;
  for (int i = 0; i < n; i++) { h ^= rec[4 + i]; h *= 1099511628211ull; }
  return h ^ (uint64_t)n;
}

// ---- DECIMAL wider than 18 digits: records are [len:int32 LE][unscaled value as BigInteger.toByteArray: big-endian, minimal
//      two's complement, 1..16 bytes] (enc/Uncompressed.scala:330-345), read into a 128-bit integer.  NVRTC needs
//      -device-int128 for them (sd_jit.cpp passes it); without it only plans free of wide DECIMALs compile ------------------
#if !defined(__CUDACC_RTC__) || defined(__CUDACC_RTC_INT128__)
#define SD_HAVE_I128 1
typedef __int128 i128;
static __device__ __noinline__ i128 dec_rec(const uint8_t* rec) {
  const int n = rec_len(rec);
  unsigned __int128 u = (unsigned __int128)(i128)(int8_t)rec[4];   // sign extension from the first byte
  for (int i = 1; i < n; i++) u = (u << 8) | rec[4 + i];
  return (i128)u;
}
// literal slot of a wide DECIMAL: 16 bytes, little-endian, 16-byte aligned in the literal pool
__device__ __forceinline__ i128 dec_lit(const uint8_t* p) {
  const uint64_t* w = reinterpret_cast<const uint64_t*>(p);
  return (i128)(((unsigned __int128)w[1] << 64) | w[0]);
}
__host__ __device__ constexpr i128 p10w(int k) { return k <= 0 ? (i128)1 : (i128)10 * p10w(k - 1); }
constexpr bool HAVE_I128 = true;
#else
constexpr bool HAVE_I128 = false;   // a plan with SLOT_MIN_DEC / SLOT_MAX_DEC slots static_asserts on it (sd_codegen.cpp)
#endif

// ---- slot (accumulator) algebra: every op is a commutative monoid over 8-byte words ------------
__device__ __forceinline__ uint64_t f2u(double d) { return (uint64_t)__double_as_longlong(d); }
__device__ __forceinline__ double u2f(uint64_t u) { return __longlong_as_double((long long)u); }

__host__ __device__ constexpr uint64_t slot_identity(int op) {
  return op == SLOT_ADD_F64 ? 0ull
       : op == SLOT_ADD_I64 ? 0ull
       : op == SLOT_MIN_I64 ? 0x7fffffffffffffffull
       : op == SLOT_MAX_I64 ? 0x8000000000000000ull
       : op == SLOT_MIN_F64 ? 0x7ff8000000000000ull   /* NaN: the greatest element of the order */
       : op == SLOT_MAX_F64 ? 0xfff0000000000000ull   /* -inf */
       : 0ull;                                         /* SLOT_MIN_STR / SLOT_MAX_STR / *_DEC: no record yet */
}
__device__ __forceinline__ uint64_t slot_combine(int op, uint64_t a, uint64_t b) {
  switch (op) {
    case SLOT_ADD_F64: return f2u(u2f(a) + u2f(b));
    case SLOT_ADD_I64: return a + b;
    case SLOT_MIN_I64: return (int64_t)b < (int64_t)a ? b : a;
    case SLOT_MAX_I64: return (int64_t)b > (int64_t)a ? b : a;
    case SLOT_MIN_F64: return f_lt(u2f(b), u2f(a)) ? b : a;
    case SLOT_MAX_F64: return f_gt(u2f(b), u2f(a)) ? b : a;
    default: {   // SLOT_MIN_STR / SLOT_MAX_STR / SLOT_MIN_DEC / SLOT_MAX_DEC: addresses of [len][bytes] records, 0 = none
      if (a == 0ull || b == 0ull || a == b) return a ? a : b;
#ifdef SD_HAVE_I128
      if (op == SLOT_MIN_DEC || op == SLOT_MAX_DEC) {
        const i128 x = dec_rec(reinterpret_cast<const uint8_t*>(b)), y = dec_rec(reinterpret_cast<const uint8_t*>(a));
        return (op == SLOT_MIN_DEC ? x < y : x > y) ? b : a;
      }
#endif
      const int c = str_cmp_recs(reinterpret_cast<const uint8_t*>(b), reinterpret_cast<const uint8_t*>(a));
      return (op == SLOT_MIN_STR ? c < 0 : c > 0) ? b : a;
    }
  }
}

// atomic version (shared or global address): used when the group table is shared by many threads
__device__ __forceinline__ void slot_atomic(int op, uint64_t* p, uint64_t v) {
  switch (op) {
    case SLOT_ADD_F64: if (v != 0ull) atomicAdd(reinterpret_cast<double*>(p), u2f(v)); break;   // x + (+0.0) == x for every running sum
    case SLOT_ADD_I64: if (v != 0ull) atomicAdd(reinterpret_cast<unsigned long long*>(p), (unsigned long long)v); break;
    case SLOT_MIN_I64: atomicMin(reinterpret_cast<long long*>(p), (long long)v); break;
    case SLOT_MAX_I64: atomicMax(reinterpret_cast<long long*>(p), (long long)v); break;
    default: {   // NaN-aware double min / max: CAS loop
      unsigned long long* a = reinterpret_cast<unsigned long long*>(p);
      unsigned long long old = *a, assumed;
      do {
        assumed = old;
        const unsigned long long want = slot_combine(op, assumed, v);
        if (want == assumed) break;
        old = atomicCAS(a, assumed, want);
      } while (old != assumed);
    }
  }
}

// ---- FIRST / LAST: (order key, value) pairs (sd_device.h SLOT_FIRST) -------------------------------------------------------
// A plan with FIRST / LAST declares NORDER > 0; only then do the loops below take the pair-aware paths, so every other plan's
// kernel is the code it always was.
template <class P, class = void> struct PlanOrders { static constexpr int N = 0; };
template <class P> struct PlanOrders<P, decltype((void)P::NORDER)> { static constexpr int N = P::NORDER; };

__device__ __forceinline__ bool order_wins(int op, uint64_t cand, uint64_t have) { return op == SLOT_FIRST ? cand < have : cand > have; }
// pair (bk, bv) into (ak, av)
__device__ __forceinline__ void order_combine(int op, uint64_t& ak, uint64_t& av, uint64_t bk, uint64_t bv) {
  if (order_wins(op, bk, ak)) { ak = bk; av = bv; }
}
// 128-bit compare-and-swap of the pair at p (16-byte aligned): returns the pair found there
template <bool SHARED>
__device__ __forceinline__ void cas_pair(uint64_t* p, uint64_t ck, uint64_t cv, uint64_t nk, uint64_t nv, uint64_t& ok, uint64_t& ov) {
  if (SHARED)
    asm volatile("{\n\t.reg .b128 c, s, r;\n\tmov.b128 c, {%2, %3};\n\tmov.b128 s, {%4, %5};\n\tatom.shared.cas.b128 r, [%6], c, s;\n\tmov.b128 {%0, %1}, r;\n\t}"
                 : "=l"(ok), "=l"(ov) : "l"(ck), "l"(cv), "l"(nk), "l"(nv), "r"((uint32_t)__cvta_generic_to_shared(p)) : "memory");
  else
    asm volatile("{\n\t.reg .b128 c, s, r;\n\tmov.b128 c, {%2, %3};\n\tmov.b128 s, {%4, %5};\n\tatom.global.cas.b128 r, [%6], c, s;\n\tmov.b128 {%0, %1}, r;\n\t}"
                 : "=l"(ok), "=l"(ov) : "l"(ck), "l"(cv), "l"(nk), "l"(nv), "l"(p) : "memory");
}
// the pair at p (shared or global memory, by SHARED) takes (k, v) when k wins.  A plain load of the key first: rows that lose --
// nearly every row of a FIRST -- issue no atomic.  The two words are read apart, so a CAS may fail on a torn expectation; it
// returns the pair as it is and the loop decides again.
template <bool SHARED>
__device__ __forceinline__ void order_atomic(int op, uint64_t* p, uint64_t k, uint64_t v) {
  uint64_t hk = *reinterpret_cast<volatile uint64_t*>(p);
  if (!order_wins(op, k, hk)) return;
  uint64_t hv = reinterpret_cast<volatile uint64_t*>(p)[1];
  for (;;) {
    uint64_t ok, ov;
    cas_pair<SHARED>(p, hk, hv, k, v, ok, ov);
    if (ok == hk && ov == hv) return;
    hk = ok; hv = ov;
    if (!order_wins(op, k, hk)) return;
  }
}
// initial word of slot op of a plan (slot_identity, and the empty order keys of a plan with FIRST / LAST)
template <class PLAN>
__device__ __forceinline__ uint64_t slot_init(int op) {
  if constexpr (PlanOrders<PLAN>::N > 0) return slot_initial(op);
  else return slot_identity(op);
}
// sv into the NSLOT entries at a (entry s at a[s * stride]) without atomics
template <class PLAN>
__device__ __forceinline__ void combine_plain(uint64_t* a, int stride, const uint64_t* sv) {
#pragma unroll
  for (int s = 0; s < PLAN::NSLOT; s++) {
    const int op = PLAN::slot_op(s);
    if (is_order_op(op)) order_combine(op, a[s * stride], a[(s + 1) * stride], sv[s], sv[s + 1]);
    else if (op != SLOT_PAIR_VAL) a[s * stride] = slot_combine(op, a[s * stride], sv[s]);
  }
}
// sv into the NSLOT entries at t with atomics (shared or global memory, by SHARED)
template <class PLAN, bool SHARED>
__device__ __forceinline__ void combine_atomic(uint64_t* t, const uint64_t* sv) {
#pragma unroll
  for (int s = 0; s < PLAN::NSLOT; s++) {
    const int op = PLAN::slot_op(s);
    if (is_order_op(op)) order_atomic<SHARED>(op, t + s, sv[s], sv[s + 1]);
    else if (op != SLOT_PAIR_VAL) slot_atomic(op, t + s, sv[s]);
  }
}

// ---- MODE_HASH: find-or-insert of a key tuple, then atomic slot updates ---------------------------------
__device__ __forceinline__ uint64_t hash_mix64(uint64_t h, uint64_t v) {
  h ^= v + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2);
  h *= 0xff51afd7ed558ccdull;
  return h ^ (h >> 33);
}
// STRMASK bit k: key k is a STRING held by reference (kc[k] = device address of its [len][bytes] record, 0 when NULL):
// hashed and compared by its bytes
__device__ __forceinline__ uint32_t ld_relaxed_u32(const uint32_t* p) { uint32_t v; asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ int64_t ld_relaxed_s64(const int64_t* p) { int64_t v; asm volatile("ld.relaxed.gpu.global.s64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v; }
// The probe / compare / publish protocol of every hash group table (the scan's and the grouping-sets roll-up's, sd_rollup.cu):
// nk keys, strmask as STRMASK above.  The scan passes compile-time constants, so its loops unroll as before.
__device__ __forceinline__ int64_t hash_probe(const HashTable& t, const int64_t* kc, uint32_t knull, int nk, uint32_t strmask) {
  uint64_t h = 0x2545f4914f6cdd1dull ^ knull;
#pragma unroll
  for (int k = 0; k < nk; k++) {
    if ((strmask >> k) & 1u) h = hash_mix64(h, kc[k] ? str_hash_rec(reinterpret_cast<const uint8_t*>(kc[k])) : 0ull);
    else h = hash_mix64(h, (uint64_t)kc[k]);
  }
  uint32_t pos = (uint32_t)h & t.mask;
  for (uint32_t probe = 0; probe < t.max_probe; probe++, pos = (pos + 1) & t.mask) {
    uint32_t st = *reinterpret_cast<volatile uint32_t*>(&t.state[pos]);
    if (st == 0u) {
      st = atomicCAS(&t.state[pos], 0u, 1u);
      if (st == 0u) {   // we own the entry: publish the key, then mark it full
#pragma unroll
        for (int k = 0; k < nk; k++) t.keys[(size_t)pos * nk + k] = kc[k];
        t.knull[pos] = knull;
        __threadfence();
        *reinterpret_cast<volatile uint32_t*>(&t.state[pos]) = 2u;
        atomicAdd(t.count, 1u);
        return pos;
      }
    }
    while (st == 1u) { __nanosleep(20); st = *reinterpret_cast<volatile uint32_t*>(&t.state[pos]); }   // writer in flight
    // The entry is published: state 2 was stored after the key, with a fence in between (writer side above).  Reader side without
    // a fence (__threadfence() here was a MEMBAR.SC.GPU + an L1 invalidate PER ROW: the largest stall of the hash kernels):
    // strong (L1-bypassing) loads whose ADDRESS depends on the state value just read, so they are issued after it returned.
    const size_t dep = (size_t)(st - 2u);   // 0; not known to the compiler
    bool same = ld_relaxed_u32(&t.knull[pos + dep]) == knull;
#pragma unroll
    for (int k = 0; k < nk; k++) {
      const int64_t have = ld_relaxed_s64(&t.keys[(size_t)pos * nk + k + dep]);
      if ((strmask >> k) & 1u) same = same && (have == kc[k] || (have && kc[k] && str_eq_recs(reinterpret_cast<const uint8_t*>(have), reinterpret_cast<const uint8_t*>(kc[k]))));
      else same = same && have == kc[k];
    }
    if (same) return pos;
  }
  atomicExch(t.overflow, 1u);
  return -1;
}
template <int NK, uint32_t STRMASK>
__device__ __forceinline__ int64_t hash_find_or_insert(const HashTable& t, const int64_t* kc, uint32_t knull) {
  return hash_probe(t, kc, knull, NK, STRMASK);
}

// ---- moment aggregates: sums S_j = sum (x - K)^j around one shift K per group ---------------------------------------------
// A plan with STDDEV / VARIANCE / SKEWNESS / KURTOSIS declares NSHIFT > 0 and, per shift i, order(i) and pow_slot(i, j) for
// j = 1..order(i).  Its slots() leaves the row's candidate K in the S_1 slot (shift_cand(x), or SHIFT_EMPTY when x is NULL);
// apply_shifts turns it into the row's contributions once the group's K (sd_device.h SHIFT_EMPTY) is known.  K is a value of the group, so the host's conversion to central moments loses digits to
// ((mean - K) / sigma)^order, not to (mean / sigma)^order as raw power sums would.
template <class P, class = void> struct PlanShifts { static constexpr int N = 0; };
template <class P> struct PlanShifts<P, decltype((void)P::NSHIFT)> { static constexpr int N = P::NSHIFT; };
// COVAR_POP / COVAR_SAMP / CORR: NPAIR > 0 cross terms S_xy = sum (x - Kx)(y - Ky), each over two of the shifts above
// (pair_shift(q, 0) = x, pair_shift(q, 1) = y; the squares CORR needs are those shifts' order-2 sums) into slot pair_slot(q)
template <class P, class = void> struct PlanPairs { static constexpr int N = 0; };
template <class P> struct PlanPairs<P, decltype((void)P::NPAIR)> { static constexpr int N = P::NPAIR; };

__device__ __forceinline__ uint64_t shift_cand(double x) { return x != x ? 0x7ff8000000000000ull : f2u(x); }
// the group's K in the word at p (beside the running result or the hash entry), claimed with `cand` while still SHIFT_EMPTY
__device__ __forceinline__ uint64_t shift_claim(uint64_t* p, uint64_t cand) {
  uint64_t k;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(k) : "l"(p) : "memory");
  if (k == SHIFT_EMPTY) {
    const unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long*>(p), SHIFT_EMPTY, cand);
    k = old == SHIFT_EMPTY ? cand : (uint64_t)old;
  }
  return k;
}
// kof(i, cand) -> the group's K of shift i
template <class PLAN, class KOf>
__device__ __forceinline__ void apply_shifts(uint64_t* sv, KOf&& kof) {
  constexpr int NP = PlanPairs<PLAN>::N;
  double dv[NP > 0 ? PLAN::NSHIFT : 1];   // x - K per shift (0 for a NULL input), kept for the cross terms
  (void)dv;
#pragma unroll
  for (int i = 0; i < PLAN::NSHIFT; i++) {
    const uint64_t cand = sv[PLAN::pow_slot(i, 1)];
    if constexpr (NP > 0) dv[i] = 0.0;
    if (cand == SHIFT_EMPTY) { sv[PLAN::pow_slot(i, 1)] = 0ull; continue; }   // NULL input: its sums stay 0
    const double d = u2f(cand) - u2f(kof(i, cand));
    if constexpr (NP > 0) dv[i] = d;
    double pw = d;
#pragma unroll
    for (int j = 1; j <= 4; j++) {
      if (j <= PLAN::order(i)) sv[PLAN::pow_slot(i, j)] = f2u(pw);
      pw *= d;
    }
  }
  if constexpr (NP > 0) {
#pragma unroll
    for (int q = 0; q < NP; q++) sv[PLAN::pair_slot(q)] = f2u(dv[PLAN::pair_shift(q, 0)] * dv[PLAN::pair_shift(q, 1)]);
  }
}

// ---- loads ------------------------------------------------------------------------------------
template <class T> __device__ __forceinline__ T ld_at(const uint8_t* base, int64_t k) {
  return *reinterpret_cast<const T*>(base + k * (int64_t)sizeof(T));
}
// RLE records are only naturally aligned to their 4-byte run length: assemble wider values bytewise
template <class T> __device__ __forceinline__ T ld_unaligned(const uint8_t* p) {
  T v;
  uint8_t* o = reinterpret_cast<uint8_t*>(&v);
#pragma unroll
  for (int i = 0; i < (int)sizeof(T); i++) o[i] = p[i];
  return v;
}
__device__ __forceinline__ int lower_bound_i32(const int32_t* a, int lo, int hi, int32_t x) {
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (a[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// k-th stored (non-null) value of a column body.  Restates the decoder read methods:
// Uncompressed (enc/Uncompressed.scala:74-98), Dictionary/BigDictionary
// (enc/DictionaryEncoding.scala:118-137,148-166), BooleanBitSet (enc/BooleanBitSetEncoding.scala:57-59),
// RunLength via host-built run-end prefix (enc/RunLengthEncoding.scala:112-172).
template <int KIND>
__device__ __forceinline__ typename KindT<KIND>::T decode_value(const uint8_t* data, const uint8_t* dict,
                                                                const int32_t* run_ends, int enc, int nruns, int64_t k) {
  typedef typename KindT<KIND>::T T;
  if (enc == ENC_UNCOMPRESSED) {
    if (KIND == K_BOOL) return (T)(data[k] == 1);
    return ld_at<T>(data, k);
  }
  if (enc == ENC_DICTIONARY || enc == ENC_BIG_DICTIONARY || enc == ENC_STR_RAW) {
    int idx = enc == ENC_DICTIONARY ? (int)ld_at<int16_t>(data, k) : ld_at<int32_t>(data, k);   // ENC_STR_RAW: record position
    if (KIND == K_CODE) return (T)idx;
    return ld_at<T>(dict, idx);
  }
  if (enc == ENC_BOOLEAN_BITSET) return (T)((ld_at<uint64_t>(data, k >> 6) >> (k & 63)) & 1);
  // ENC_RUN_LENGTH: first run whose exclusive end exceeds k
  int run = lower_bound_i32(run_ends, 0, nruns, (int32_t)k + 1);
  if (KIND == K_CODE) return (T)ld_at<int32_t>(dict, run);
  return ld_unaligned<T>(data + (int64_t)run * (sizeof(T) + 4));
}

// value of an update-delta entry; K_CODE entries are translated to the batch's unified code space
template <int KIND>
__device__ __forceinline__ typename KindT<KIND>::T decode_delta_value(const DevDelta& d, int64_t k) {
  typedef typename KindT<KIND>::T T;
  if (KIND == K_CODE) {
    int idx = d.enc == ENC_DICTIONARY ? (int)ld_at<int16_t>(d.data, k) : ld_at<int32_t>(d.data, k);
    return (T)ld_at<int32_t>(d.dict, idx);
  }
  return decode_value<KIND>(d.data, d.dict, nullptr, d.enc, 0, k);
}

// Out-of-line helpers for the per-row paths.  They are instantiated once per value kind instead of once per
// (column, row-of-thread), which keeps the NVRTC compile of a plan short (the inlined form made up two thirds of
// Q1's 10 s compile) and costs nothing on the staged paths that never call them.
//
// base value #k of a column in any encoding but the directly addressable uncompressed one
template <int KIND>
__device__ __noinline__ typename KindT<KIND>::T decode_value_slow(const uint8_t* data, const uint8_t* dict, const int32_t* run_ends,
                                                                  int enc, int nruns, int64_t k) {
  return decode_value<KIND>(data, dict, run_ends, enc, nruns, k);
}
template <int KIND>
__device__ __forceinline__ typename KindT<KIND>::T decode_value_any(const uint8_t* data, const uint8_t* dict, const int32_t* run_ends,
                                                                    int enc, int nruns, int64_t k) {
  typedef typename KindT<KIND>::T T;
  if (enc == ENC_UNCOMPRESSED) {
    if (KIND == K_BOOL) return (T)(data[k] == 1);
    return ld_at<T>(data, k);
  }
  return decode_value_slow<KIND>(data, dict, run_ends, enc, nruns, k);
}
// value of row `i` from the column's update deltas (the row's bit is set in the tile's update bitmap, so one of the
// two deltas holds it); the depth-0 delta wins on equal position (enc/UpdatedColumnDecoder.scala:95-104); null
// bits index the relative entry (enc/ColumnDeltaDecoder.scala:77-83).  r0..r3 = [lo, hi) of delta0 / delta1
// positions inside the tile.
template <int KIND>
__device__ __noinline__ typename KindT<KIND>::T delta_lookup(const DevDelta* d0, const DevDelta* d1, int r0, int r1, int r2, int r3,
                                                             int32_t i, int null_code, bool* out_null) {
  typedef typename KindT<KIND>::T T;
  const DevDelta* d = d0;
  int j = -1;
  if (d) {
    int q = lower_bound_i32(d->positions, r0, r1, i);
    if (q < r1 && d->positions[q] == i) j = q;
  }
  if (j < 0) {
    d = d1;
    j = lower_bound_i32(d->positions, r2, r3, i);
  }
  int64_t k = j;
  bool isnull = false;
  if (d->nulls) {
    const int w = j >> 6;
    const uint64_t word = w < d->nwords ? d->nulls[w] : 0ull;
    isnull = (word >> (j & 63)) & 1ull;
    int before = __popcll(word & ((1ull << (j & 63)) - 1ull));
    for (int x = 0; x < w && x < d->nwords; x++) before += __popcll(d->nulls[x]);
    k = j - before;
  }
  *out_null = isnull;
  if (!isnull) return decode_delta_value<KIND>(*d, k);
  return KIND == K_CODE ? (T)null_code : (T)0;   // NULL code (ColumnTableScan.scala:706-716)
}

// ---- per-thread registers of one tile -----------------------------------------------------------
template <class PLAN, int C>
struct ColRegs {
  typedef typename KindT<PLAN::kind(C)>::T T;
  T v[PLAN::RPT];
  uint32_t nullmask;   // bit r: row r of this thread is NULL in column C
};
template <class PLAN, class S> struct AllCols;
template <class PLAN, int... Cs> struct AllCols<PLAN, Seq<Cs...>> : ColRegs<PLAN, Cs>... {};

template <class PLAN>
struct TileSmem {
  static constexpr int TILE_ROWS = THREADS * PLAN::RPT;
  static constexpr int TILE_WORDS = TILE_ROWS / 64;
  uint32_t delbits[TILE_ROWS / 32];
  uint32_t updbits[PLAN::NC > 0 ? PLAN::NC : 1][TILE_ROWS / 32];
  int32_t wprefix[PLAN::NC > 0 ? PLAN::NC : 1][TILE_WORDS];
  int32_t drange[PLAN::NC > 0 ? PLAN::NC : 1][4];   // per column: [lo, hi) of delta0 and delta1 positions inside the tile
  int32_t delrange[2];                               // [lo, hi) of the delete positions inside the tile
  // overlay path: per-warp cursors into the sorted delete / delta positions (a warp's 64-row segments are visited in
  // ascending order inside a chunk, so every list is walked once, linearly, by each warp on its own -- no CTA barrier)
  int32_t wdel[THREADS / 32];
  int32_t wcur[PLAN::NC > 0 ? PLAN::NC : 1][THREADS / 32][2];
};

// row r of a thread within tile: pair u = r/2 at tile + u*2*THREADS + 2*tid + (r&1)
__device__ __forceinline__ int row_in_tile(int r) { return (r >> 1) * 2 * THREADS + 2 * (int)threadIdx.x + (r & 1); }

// ---- fast path: coalesced vector loads ------------------------------------------------------------
template <class PLAN, int C>
__device__ __forceinline__ void load_col_fast(const DevCol& col, int64_t tile_start, ColRegs<PLAN, C>& regs) {
  typedef typename KindT<PLAN::kind(C)>::T T;
  constexpr int K = PLAN::kind(C);
  regs.nullmask = 0;
#pragma unroll
  for (int u = 0; u < PLAN::RPT / 2; u++) {
    const int64_t p = tile_start + u * 2 * THREADS + 2 * (int)threadIdx.x;   // even row index
    if (K == K_CODE) {
      if (col.enc == ENC_DICTIONARY) {
        uint32_t x = __ldcs(reinterpret_cast<const uint32_t*>(col.data + p * 2));
        regs.v[2 * u] = (T)(int16_t)(x & 0xffffu);
        regs.v[2 * u + 1] = (T)(int16_t)(x >> 16);
      } else {
        int2 x = __ldcs(reinterpret_cast<const int2*>(col.data + p * 4));
        regs.v[2 * u] = (T)x.x;
        regs.v[2 * u + 1] = (T)x.y;
      }
    } else if (sizeof(T) == 8) {
      longlong2 x = __ldcs(reinterpret_cast<const longlong2*>(col.data + p * 8));
      regs.v[2 * u] = K == K_F64 ? (T)__longlong_as_double(x.x) : (T)x.x;
      regs.v[2 * u + 1] = K == K_F64 ? (T)__longlong_as_double(x.y) : (T)x.y;
    } else if (sizeof(T) == 4) {
      int2 x = __ldcs(reinterpret_cast<const int2*>(col.data + p * 4));
      regs.v[2 * u] = K == K_F32 ? (T)__int_as_float(x.x) : (T)x.x;
      regs.v[2 * u + 1] = K == K_F32 ? (T)__int_as_float(x.y) : (T)x.y;
    } else if (sizeof(T) == 2) {
      uint32_t x = __ldcs(reinterpret_cast<const uint32_t*>(col.data + p * 2));
      regs.v[2 * u] = (T)(int16_t)(x & 0xffffu);
      regs.v[2 * u + 1] = (T)(int16_t)(x >> 16);
    } else {
      uint16_t x = __ldcs(reinterpret_cast<const uint16_t*>(col.data + p));
      regs.v[2 * u] = K == K_BOOL ? (T)((x & 0xff) == 1) : (T)(int8_t)(x & 0xff);
      regs.v[2 * u + 1] = K == K_BOOL ? (T)((x >> 8) == 1) : (T)(int8_t)(x >> 8);
    }
  }
}

// ---- general path: nulls, deltas, every encoding -------------------------------------------------
template <class PLAN, int C>
__device__ __forceinline__ void load_col_general(const DevCol& col, int tile, int64_t tile_start, int num_rows,
                                                 const TileSmem<PLAN>& sm, ColRegs<PLAN, C>& regs) {
  typedef typename KindT<PLAN::kind(C)>::T T;
  constexpr int K = PLAN::kind(C);
  regs.nullmask = 0;
  const bool has_delta = col.delta0 != nullptr || col.delta1 != nullptr;
  // nulls before this tile: host prefix per NULL_PREFIX_ROWS rows (+ the words in between for big tiles
  // are covered because the prefix index is taken at the tile start and tiles are multiples of it)
  const int tile_nulls = col.tile_nulls ? col.tile_nulls[tile_start / NULL_PREFIX_ROWS] : 0;
#pragma unroll
  for (int r = 0; r < PLAN::RPT; r++) {
    const int li = row_in_tile(r);
    const int64_t i = tile_start + li;
    T v = (T)0;
    bool isnull = false;
    if (i < num_rows) {
      const bool upd = has_delta && ((sm.updbits[C][li >> 5] >> (li & 31)) & 1u);
      if (!upd) {   // base value: k = ordinal - nulls before it (ColumnTableScan.scala:794-815)
        int64_t k = i;
        if (col.nulls) {
          const int w = (int)(i >> 6);
          const uint64_t word = w < col.nwords ? col.nulls[w] : 0ull;
          isnull = (word >> (i & 63)) & 1ull;
          k = i - (tile_nulls + sm.wprefix[C][li >> 6] + __popcll(word & ((1ull << (i & 63)) - 1ull)));
        }
        if (!isnull) v = decode_value_any<K>(col.data, col.dict, col.run_ends, col.enc, col.nruns, k);
      } else {
        v = delta_lookup<K>(col.delta0, col.delta1, sm.drange[C][0], sm.drange[C][1], sm.drange[C][2], sm.drange[C][3],
                            (int32_t)i, col.dict_n, &isnull);
      }
      if (isnull && K == K_CODE) v = (T)col.dict_n;   // NULL code (ColumnTableScan.scala:706-716)
    }
    regs.v[r] = v;
    regs.nullmask |= (isnull ? 1u : 0u) << r;
  }
}

// value of entry j of an update delta (null bits index the relative entry, enc/ColumnDeltaDecoder.scala:77-83)
template <int KIND>
__device__ __noinline__ typename KindT<KIND>::T delta_value_at(const DevDelta* d, int j, int null_code, bool* out_null) {
  typedef typename KindT<KIND>::T T;
  int64_t k = j;
  bool isnull = false;
  if (d->nulls) {
    const int w = j >> 6;
    const uint64_t word = w < d->nwords ? d->nulls[w] : 0ull;
    isnull = (word >> (j & 63)) & 1ull;
    int before = __popcll(word & ((1ull << (j & 63)) - 1ull));
    for (int x = 0; x < w && x < d->nwords; x++) before += __popcll(d->nulls[x]);
    k = j - before;
  }
  *out_null = isnull;
  if (!isnull) return decode_delta_value<KIND>(*d, k);
  return KIND == K_CODE ? (T)null_code : (T)0;
}

// The entries of the ascending list `pos` that fall into the 64-row segment [a, a + 64), found by one warp on its own:
// -> bit mask (bit = position - a) and, in *first, the list index of the lowest one; *cur is the warp's cursor into the
// list (everything below it lies before this warp's previous segments) and is advanced past the segment.  One or two
// coalesced 32-entry loads, ballots and warp OR-reductions; no shared memory, no barrier.
__device__ __forceinline__ uint64_t warp_segment_mask(const int32_t* pos, int n, int32_t a, int& cur, int lane, int* first) {
  for (;;) {   // skip what belongs to other warps' segments
    const int idx = cur + lane;
    const int32_t p = idx < n ? __ldg(pos + idx) : 0x7fffffff;
    const int c = __popc(__ballot_sync(0xffffffffu, p < a));
    cur += c;
    if (c < 32) break;
  }
  *first = cur;
  uint64_t mask = 0;
  for (;;) {
    const int idx = cur + lane;
    const int32_t p = idx < n ? __ldg(pos + idx) : 0x7fffffff;
    const bool in = p < a + 64;
    const int bit = in ? (int)(p - a) : 0;
    const unsigned lo = __reduce_or_sync(0xffffffffu, (in && bit < 32) ? (1u << bit) : 0u);
    const unsigned hi = __reduce_or_sync(0xffffffffu, (in && bit >= 32) ? (1u << (bit - 32)) : 0u);
    mask |= (uint64_t)lo | ((uint64_t)hi << 32);
    const int c = __popc(__ballot_sync(0xffffffffu, in));
    cur += c;
    if (c < 32) break;
  }
  return mask;
}
static __device__ __noinline__ int warp_cursor_init(const int32_t* pos, int n, int32_t a) { return lower_bound_i32(pos, 0, n, a); }

// overlay of one column, per warp: rows whose position is in the depth-0 delta take that value, else the depth-1 delta's
// (enc/UpdatedColumnDecoder.scala:95-104)
template <class PLAN, int C>
__device__ __forceinline__ void warp_overlay_col(const DevCol& col, int64_t tile_start, bool first_tile, TileSmem<PLAN>& sm, ColRegs<PLAN, C>& regs) {
  typedef typename KindT<PLAN::kind(C)>::T T;
  constexpr int K = PLAN::kind(C);
  const DevDelta *d0 = col.delta0, *d1 = col.delta1;
  if (!(d0 || d1)) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int32_t a0 = (int32_t)tile_start + warp * 64;
  int cur0 = 0, cur1 = 0;
  if (first_tile) {
    if (d0) cur0 = warp_cursor_init(d0->positions, d0->n, a0);
    if (d1) cur1 = warp_cursor_init(d1->positions, d1->n, a0);
  } else { cur0 = sm.wcur[C][warp][0]; cur1 = sm.wcur[C][warp][1]; }
#pragma unroll
  for (int u = 0; u < PLAN::RPT / 2; u++) {
    const int32_t a = a0 + u * 2 * THREADS;
    int f0 = 0, f1 = 0;
    const uint64_t m0 = d0 ? warp_segment_mask(d0->positions, d0->n, a, cur0, lane, &f0) : 0ull;
    const uint64_t m1 = d1 ? warp_segment_mask(d1->positions, d1->n, a, cur1, lane, &f1) : 0ull;
    if ((m0 | m1) == 0ull) continue;
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int r = 2 * u + h, bit = 2 * lane + h;
      const uint64_t below = (1ull << bit) - 1ull;
      bool isnull = false;
      if ((m0 >> bit) & 1ull) {
        regs.v[r] = delta_value_at<K>(d0, f0 + __popcll(m0 & below), col.dict_n, &isnull);
        regs.nullmask = (regs.nullmask & ~(1u << r)) | ((isnull ? 1u : 0u) << r);
      } else if ((m1 >> bit) & 1ull) {
        regs.v[r] = delta_value_at<K>(d1, f1 + __popcll(m1 & below), col.dict_n, &isnull);
        regs.nullmask = (regs.nullmask & ~(1u << r)) | ((isnull ? 1u : 0u) << r);
      }
    }
  }
  __syncwarp();
  if (lane == 0) { sm.wcur[C][warp][0] = cur0; sm.wcur[C][warp][1] = cur1; }
  __syncwarp();
}
template <class PLAN, int... Cs>
__device__ __forceinline__ void warp_overlay_all(const DevBatch<PLAN::NC>& b, int64_t tile_start, bool first_tile, TileSmem<PLAN>& sm,
                                                 AllCols<PLAN, Seq<Cs...>>& regs, uint32_t& live, Seq<Cs...>) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (b.deletes) {   // delete mask (enc/ColumnDeleteDecoder.scala:49-55)
    const int32_t a0 = (int32_t)tile_start + warp * 64;
    int cur = first_tile ? warp_cursor_init(b.deletes, b.num_deletes, a0) : sm.wdel[warp];
#pragma unroll
    for (int u = 0; u < PLAN::RPT / 2; u++) {
      int f;
      const uint64_t m = warp_segment_mask(b.deletes, b.num_deletes, a0 + u * 2 * THREADS, cur, lane, &f);
      if ((m >> (2 * lane)) & 1ull) live &= ~(1u << (2 * u));
      if ((m >> (2 * lane + 1)) & 1ull) live &= ~(1u << (2 * u + 1));
    }
    __syncwarp();
    if (lane == 0) sm.wdel[warp] = cur;
    __syncwarp();
  }
  int dummy[] = {0, (warp_overlay_col<PLAN, Cs>(b.cols[Cs], tile_start, first_tile, sm, static_cast<ColRegs<PLAN, Cs>&>(regs)), 0)...};
  (void)dummy;
}

// fast + overlay path: the base values were loaded by the staged vector path; rows whose bit is set in the tile's
// update bitmap are replaced by their delta value (depth 0 wins), exactly like the general path does
template <class PLAN, int C>
__device__ __forceinline__ void overlay_col(const DevCol& col, int64_t tile_start, int num_rows, const TileSmem<PLAN>& sm,
                                            ColRegs<PLAN, C>& regs) {
  typedef typename KindT<PLAN::kind(C)>::T T;
  constexpr int K = PLAN::kind(C);
  if (!(col.delta0 || col.delta1)) return;
#pragma unroll
  for (int r = 0; r < PLAN::RPT; r++) {
    const int li = row_in_tile(r);
    const int64_t i = tile_start + li;
    if (i >= num_rows || !((sm.updbits[C][li >> 5] >> (li & 31)) & 1u)) continue;
    bool isnull = false;
    const T v = delta_lookup<K>(col.delta0, col.delta1, sm.drange[C][0], sm.drange[C][1], sm.drange[C][2], sm.drange[C][3],
                                (int32_t)i, col.dict_n, &isnull);
    regs.v[r] = v;
    regs.nullmask = (regs.nullmask & ~(1u << r)) | ((isnull ? 1u : 0u) << r);
  }
}
template <class PLAN, int... Cs>
__device__ __forceinline__ void overlay_all(const DevBatch<PLAN::NC>& b, int64_t tile_start, const TileSmem<PLAN>& sm,
                                            AllCols<PLAN, Seq<Cs...>>& regs, Seq<Cs...>) {
  int dummy[] = {0, (overlay_col<PLAN, Cs>(b.cols[Cs], tile_start, b.num_rows, sm, static_cast<ColRegs<PLAN, Cs>&>(regs)), 0)...};
  (void)dummy;
}

// [lo, hi) of the sorted `positions` that fall into [ts, te), found by one warp: `lo` continues from the previous
// tile's `hi` (tiles of a chunk are visited in order; first >= 0) or comes from a binary search; `hi` is found 32
// entries at a time with a ballot (a 1024-row tile rarely holds more than a handful of updated / deleted rows)
__device__ __forceinline__ void warp_find_range(const int32_t* positions, int n, int32_t ts, int32_t te, int first, int lane, int* out_lo, int* out_hi) {
  int lo = first >= 0 ? first : lower_bound_i32(positions, 0, n, ts);
  int hi = lo;
  for (;;) {
    const int idx = hi + lane;
    const unsigned m = __ballot_sync(0xffffffffu, idx < n && positions[idx] < te);
    const int c = __popc(m);
    hi += c;
    if (c < 32) break;
  }
  *out_lo = lo;
  *out_hi = hi;
}
// one copy for all columns and plans (out of line: see decode_value_slow)
static __device__ __noinline__ void find_delta_ranges(const DevDelta* d0, const DevDelta* d1, int32_t ts, int32_t te, bool first_tile, int32_t* drange, int lane) {
#pragma unroll
  for (int dd = 0; dd < 2; dd++) {
    const DevDelta* d = dd == 0 ? d0 : d1;
    int lo = 0, hi = 0;
    const int first = first_tile ? -1 : drange[2 * dd + 1];
    if (d) warp_find_range(d->positions, d->n, ts, te, first, lane, &lo, &hi);
    __syncwarp();   // every lane has read the previous tile's cursor before lane 0 replaces it
    if (lane == 0) { drange[2 * dd] = lo; drange[2 * dd + 1] = hi; }
  }
}
static __device__ __noinline__ void find_delete_range(const int32_t* deletes, int n, int32_t ts, int32_t te, bool first_tile, int32_t* delrange, int lane) {
  int lo, hi;
  const int first = first_tile ? -1 : delrange[1];
  warp_find_range(deletes, n, ts, te, first, lane, &lo, &hi);
  __syncwarp();
  if (lane == 0) { delrange[0] = lo; delrange[1] = hi; }
}
template <class PLAN, int C>
__device__ __forceinline__ void find_col_ranges(const DevCol& col, int64_t tile_start, bool first_tile, TileSmem<PLAN>& sm, int lane) {
  if (!(col.delta0 || col.delta1)) return;
  const int32_t ts = (int32_t)tile_start;
  find_delta_ranges(col.delta0, col.delta1, ts, ts + TileSmem<PLAN>::TILE_ROWS, first_tile, sm.drange[C], lane);
}
template <class PLAN, int... Cs>
__device__ __forceinline__ void find_all_ranges(const DevBatch<PLAN::NC>& b, int64_t tile_start, bool first_tile, TileSmem<PLAN>& sm, int lane, Seq<Cs...>) {
  int dummy[] = {0, (find_col_ranges<PLAN, Cs>(b.cols[Cs], tile_start, first_tile, sm, lane), 0)...};
  (void)dummy;
  if (b.deletes)
    find_delete_range(b.deletes, b.num_deletes, (int32_t)tile_start, (int32_t)tile_start + TileSmem<PLAN>::TILE_ROWS, first_tile, sm.delrange, lane);
}

// tile preparation for the general path: null-word prefix sums, delete / update bitmaps
template <int TILE_WORDS>
__device__ __noinline__ void prep_col_words(const DevCol* colp, int64_t tile_start, int32_t* wprefix, uint32_t* updbits, const int32_t* drange) {
  const DevCol& col = *colp;
  const int tid = threadIdx.x;
  if (col.nulls && tid < TILE_WORDS) {   // warp 0, lanes 0..TILE_WORDS-1: exclusive scan of per-word popcounts
    const int w = (int)(tile_start >> 6) + tid;
    const int pc = w < col.nwords ? __popcll(col.nulls[w]) : 0;
    int inc = pc;
#pragma unroll
    for (int d = 1; d < TILE_WORDS; d <<= 1) {
      int t = __shfl_up_sync((TILE_WORDS >= 32 ? 0xffffffffu : ((1u << TILE_WORDS) - 1u)), inc, d, TILE_WORDS);
      if (tid >= d) inc += t;
    }
    wprefix[tid] = inc - pc;
  }
  if (col.delta0 || col.delta1) {   // scatter the tile's updated positions (ranges found by find_all_ranges) into the bitmap
    const int32_t ts = (int32_t)tile_start;
#pragma unroll
    for (int dd = 0; dd < 2; dd++) {
      const DevDelta* d = dd == 0 ? col.delta0 : col.delta1;
      if (d) {
        const int lo = drange[2 * dd], hi = drange[2 * dd + 1];
        for (int j = lo + tid; j < hi; j += THREADS) {
          const int li = d->positions[j] - ts;
          atomicOr(&updbits[li >> 5], 1u << (li & 31));
        }
      }
    }
  }
}
template <class PLAN, int C>
__device__ __forceinline__ void prep_col_general(const DevCol& col, int64_t tile_start, TileSmem<PLAN>& sm) {
  if (col.nulls || col.delta0 || col.delta1) prep_col_words<TileSmem<PLAN>::TILE_WORDS>(&col, tile_start, sm.wprefix[C], sm.updbits[C], sm.drange[C]);
}

template <class PLAN, int... Cs>
__device__ __forceinline__ void load_all_fast(const DevBatch<PLAN::NC>& b, int64_t tile_start,
                                              AllCols<PLAN, Seq<Cs...>>& regs, Seq<Cs...>) {
  int dummy[] = {0, (load_col_fast<PLAN, Cs>(b.cols[Cs], tile_start, static_cast<ColRegs<PLAN, Cs>&>(regs)), 0)...};
  (void)dummy;
}
#ifndef SD_EXP_VERIFY
#define SD_EXP_VERIFY 0
#endif
// SD_EXP_VERIFY (diagnostic builds only): the staged copy of a tile against the same rows read straight from global memory
template <class PLAN, int C>
__device__ __forceinline__ void verify_col(const ColRegs<PLAN, C>& a, const ColRegs<PLAN, C>& b, uint32_t live, int64_t tile_start, int stage,
                                           unsigned long long* counters, const DevCol& col, int nstages, int num_rows, uint32_t* hist, int* any) {
  typedef typename KindT<PLAN::kind(C)>::T T;
#pragma unroll
  for (int r = 0; r < PLAN::RPT; r++) {
    if (!((live >> r) & 1u)) continue;
    unsigned long long x = 0, y = 0;
    memcpy(&x, &a.v[r], sizeof(a.v[r]));
    memcpy(&y, &b.v[r], sizeof(b.v[r]));
    if (x != y) {
      // whose value is it?  the stage's previous / next occupant inside the same batch (k tiles back / ahead, k = nstages)
      const int64_t row = tile_start + row_in_tile(r), span = (int64_t)nstages * THREADS * PLAN::RPT;
      const T* base = reinterpret_cast<const T*>(col.data);
      unsigned long long pv = ~0ull, nv = ~0ull;
      if (row - span >= 0) { pv = 0; memcpy(&pv, &base[row - span], sizeof(T)); }
      if (row + span < num_rows) { nv = 0; memcpy(&nv, &base[row + span], sizeof(T)); }
      if (x == pv) atomicAdd(&counters[2], 1ull); else if (x == nv) atomicAdd(&counters[3], 1ull);
      atomicAdd(&counters[4], 1ull);
      if (hist) { atomicAdd(&hist[16 + (threadIdx.x >> 5)], 1u); atomicAdd(&hist[24 + ((row_in_tile(r) >> 7) & 7)], 1u); atomicAdd(&hist[32 + (C & 3)], 1u); *any = 1; }
      const unsigned long long tag = ((unsigned long long)(C + 1) << 56) | ((unsigned long long)stage << 48) | ((unsigned long long)(tile_start + row_in_tile(r)) & 0xffffffffffffull);
      if (atomicCAS(&counters[5], 0ull, tag) == 0ull) { counters[6] = x; counters[7] = y; }
    }
  }
}
template <class PLAN, int... Cs>
__device__ __forceinline__ void verify_all(const AllCols<PLAN, Seq<Cs...>>& a, const AllCols<PLAN, Seq<Cs...>>& b, uint32_t live, int64_t tile_start,
                                           int stage, unsigned long long* counters, const DevBatch<PLAN::NC>& bt, int nstages, uint32_t* hist, Seq<Cs...>) {
  int any = 0;
  int dummy[] = {0, (verify_col<PLAN, Cs>(static_cast<const ColRegs<PLAN, Cs>&>(a), static_cast<const ColRegs<PLAN, Cs>&>(b), live, tile_start, stage, counters,
                                          bt.cols[Cs], nstages, bt.num_rows, hist, &any), 0)...};
  if (hist) {
    const unsigned m = __ballot_sync(0xffffffffu, any != 0);
    if ((threadIdx.x & 31) == 0) { atomicAdd(&hist[41], 1u); if (m) atomicAdd(&hist[40], 1u); }
  }
  (void)dummy;
}
#ifndef SD_EXP_SKIP_ROWS
#define SD_EXP_SKIP_ROWS 0
#endif
#ifndef SD_EXP_SINK_GROUPS
#define SD_EXP_SINK_GROUPS 0
#endif
// SD_EXP_SKIP_ROWS (diagnostic builds only): a tile's loads end in a register sink instead of the row loop
template <class PLAN, int C>
__device__ __forceinline__ void fold_col(const ColRegs<PLAN, C>& a, uint64_t& sink) {
  sink ^= a.nullmask;
#pragma unroll
  for (int r = 0; r < PLAN::RPT; r++) {
    unsigned long long x = 0;
    memcpy(&x, &a.v[r], sizeof(a.v[r]));
    sink ^= x;
  }
}
template <class PLAN, int... Cs>
__device__ __forceinline__ void fold_all(const AllCols<PLAN, Seq<Cs...>>& a, uint64_t& sink, Seq<Cs...>) {
  int dummy[] = {0, (fold_col<PLAN, Cs>(static_cast<const ColRegs<PLAN, Cs>&>(a), sink), 0)...};
  (void)dummy;
}
template <class PLAN, int... Cs>
__device__ __forceinline__ void clear_upd_bits(const DevBatch<PLAN::NC>& b, TileSmem<PLAN>& sm, Seq<Cs...>) {
  const int tid = threadIdx.x;
  if (tid < TileSmem<PLAN>::TILE_ROWS / 32) {
    sm.delbits[tid] = 0;
    int dummy[] = {0, ((b.cols[Cs].delta0 || b.cols[Cs].delta1) ? (sm.updbits[Cs][tid] = 0, 0) : 0)...};
    (void)dummy;
  }
}
template <class PLAN, int... Cs>
__device__ __forceinline__ void prep_all_general(const DevBatch<PLAN::NC>& b, int64_t tile_start, TileSmem<PLAN>& sm, Seq<Cs...>) {
  int dummy[] = {0, (prep_col_general<PLAN, Cs>(b.cols[Cs], tile_start, sm), 0)...};
  (void)dummy;
}
template <class PLAN, int... Cs>
__device__ __forceinline__ void load_all_general(const DevBatch<PLAN::NC>& b, int tile, int64_t tile_start,
                                                 const TileSmem<PLAN>& sm, AllCols<PLAN, Seq<Cs...>>& regs, Seq<Cs...>) {
  int dummy[] = {0, (load_col_general<PLAN, Cs>(b.cols[Cs], tile, tile_start, b.num_rows, sm,
                                                static_cast<ColRegs<PLAN, Cs>&>(regs)), 0)...};
  (void)dummy;
}
template <class PLAN, int... Cs>
__device__ __forceinline__ void fill_row(const AllCols<PLAN, Seq<Cs...>>& regs, int r, typename PLAN::Row& row, Seq<Cs...>) {
  int dummy[] = {0, (row.template set<Cs>(static_cast<const ColRegs<PLAN, Cs>&>(regs).v[r],
                                          (static_cast<const ColRegs<PLAN, Cs>&>(regs).nullmask >> r) & 1u), 0)...};
  (void)dummy;
}


// ---- shared-memory ring fed by bulk async copies (TMA unit, SASS: UBLKCP) ---------------------------
// A producer thread issues one cp.async.bulk per column tile; completion is tracked by an mbarrier
// (complete_tx byte counting).  Bytes in flight are then bounded by shared memory (up to ~200 KB per
// SM), not by registers x resident warps -- which is what a pure HBM-read-bound scan needs.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* b) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(b)), "r"(parity) : "memory");
  } while (!ok);
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// consumer-only CTA barrier (the producer warp never joins it)
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(THREADS) : "memory"); }

// byte offset of column C's tile inside a stage of the verbatim layout (every column at its kind's widest element)
template <class PLAN>
__host__ __device__ constexpr int stage_col_off(int c) {
  int off = 0;
  // + 128: a column with NULLs is copied from the 16-byte boundary below its first value of the tile (<= 15 extra
  // bytes); a full 128 keeps every column's region 128-byte aligned for the bulk copies
  for (int i = 0; i < c; i++) off += THREADS * PLAN::RPT * kind_stage_width(PLAN::kind(i)) + 128;
  return off;
}
// word offset of column C's img_tab copy in the kernel's shared-memory image tables (ScanArgs.img_off) in the verbatim layout
template <class PLAN>
__host__ __device__ constexpr int img_col_off(int c) {
  int off = 0;
  for (int i = 0; i < c; i++) off += img_smem_words(PLAN::kind(i));
  return off;
}
template <class PLAN>
struct StageInfo {
  static constexpr int BYTES = stage_col_off<PLAN>(PLAN::NC);
};
// The ring layout a kernel reads (RT): the launch's (RingArgs, sized by what the launch streams: the two-CTA kernel of a
// dense group-by), or the verbatim layout as constants (every other kernel)
template <class PLAN, bool RT, int C>
__device__ __forceinline__ int stage_off(const RingArgs& r) { return RT ? r.stage_off[C] : stage_col_off<PLAN>(C); }
template <class PLAN, bool RT>
__device__ __forceinline__ int stage_size(const RingArgs& r) { return RT ? r.stage_bytes : StageInfo<PLAN>::BYTES; }
template <class PLAN, bool RT, int C>
__device__ __forceinline__ int img_col(const RingArgs& r) { return RT ? r.img_col[C] : img_col_off<PLAN>(C); }

// one bit per scan column: 32 bits for plans of <= 32 columns (the common case keeps its register budget), 64 beyond
template <bool WIDE> struct CMaskT { typedef uint32_t T; };
template <> struct CMaskT<true> { typedef uint64_t T; };
#define SD_CMASK(PLAN) typename CMaskT<(PLAN::NC > 32)>::T

// what the staged loads of one batch read, one bit per column (uniform per work item)
template <class PLAN>
struct ColModes {
  typedef SD_CMASK(PLAN) M;
  M c16;      // K_CODE column with int16 dictionary indexes (else int32)
  M img;      // the column's scan image (DevCol.img) instead of its verbatim values
  M w1;       // image width 1 (else 2)
};
__host__ __device__ constexpr bool kind_has_image(int k) { return k != K_BOOL && k != K_I8; }

// element width of column C in this batch (dictionary indexes are int16 or int32; images 1 or 2 bytes)
template <class PLAN, int C>
__device__ __forceinline__ int col_width(const ColModes<PLAN>& cm) {
  if (kind_has_image(PLAN::kind(C)) && ((cm.img >> C) & 1)) return ((cm.w1 >> C) & 1) ? 1 : 2;
  return PLAN::kind(C) == K_CODE ? (((cm.c16 >> C) & 1) ? 2 : 4) : (int)sizeof(typename KindT<PLAN::kind(C)>::T);
}

// per-chunk copy of the descriptor fields the producer needs (with the SM's shared memory carved out for the ring
// the L1 is tiny: re-reading them from the batch descriptor for every tile costs an L2 round trip each)
template <int NC>
struct ProducerCols {
  const uint8_t* data[NC > 0 ? NC : 1];
  const int32_t* tile_nulls[NC > 0 ? NC : 1];
};
template <class PLAN, int... Cs>
__device__ __forceinline__ void load_producer_cols(const DevBatch<PLAN::NC>& b, const ColModes<PLAN>& cm, ProducerCols<PLAN::NC>& pc, Seq<Cs...>) {
  int dummy[] = {0, (pc.data[Cs] = ((cm.img >> Cs) & 1) ? b.cols[Cs].img : b.cols[Cs].data,
                     pc.tile_nulls[Cs] = PLAN::col_nullable(Cs) ? b.cols[Cs].tile_nulls : nullptr, 0)...};
  (void)dummy;
}

// source range of column C's values for the tile [tile_start, tile_start + rows): without NULLs value index == row
// ordinal; with NULLs the tile's stored values are [tile_start - nulls_before(tile_start), ... ) and their count is
// rows - nulls_in_tile, both from the host-computed prefix (one entry per NULL_PREFIX_ROWS rows)
template <class PLAN, int C>
__device__ __forceinline__ void col_copy_range(const int32_t* tile_nulls, const ColModes<PLAN>& cm, int64_t tile_start, int rows, int64_t* src_off, uint32_t* bytes) {
  const int w = col_width<PLAN, C>(cm);
  int64_t first = tile_start;
  int cnt = rows;
  if (PLAN::col_nullable(C) && tile_nulls) {
    const int n0 = tile_nulls[tile_start / NULL_PREFIX_ROWS];
    const int n1 = tile_nulls[(tile_start + rows + NULL_PREFIX_ROWS - 1) / NULL_PREFIX_ROWS];
    first = tile_start - n0;
    cnt = rows - (n1 - n0);
  }
  const int64_t off = first * w;
  *src_off = off & ~int64_t(15);
  *bytes = cnt > 0 ? (uint32_t)(((off & 15) + (int64_t)cnt * w + 15) & ~int64_t(15)) : 0u;   // buffers are padded: over-reading is safe
}
template <class PLAN, bool RT, int... Cs>
__device__ __forceinline__ void issue_tile_copies(const RingArgs& a, const ProducerCols<PLAN::NC>& pc, const ColModes<PLAN>& cm, int64_t tile_start, int rows, uint8_t* stage, uint64_t* bar, Seq<Cs...>) {
  int64_t off[PLAN::NC > 0 ? PLAN::NC : 1];
  uint32_t bytes[PLAN::NC > 0 ? PLAN::NC : 1];
  uint32_t total = 0;
  int d0[] = {0, (col_copy_range<PLAN, Cs>(pc.tile_nulls[Cs], cm, tile_start, rows, &off[Cs], &bytes[Cs]), total += bytes[Cs], 0)...};
  (void)d0;
  mbar_expect_tx(bar, total);
  int d1[] = {0, ((!PLAN::col_nullable(Cs) || bytes[Cs]) ? (bulk_g2s(stage + stage_off<PLAN, RT, Cs>(a), pc.data[Cs] + off[Cs], bytes[Cs], bar), 0) : 0)...};
  (void)d1;
}

// value of image code x: dictionary entry (floating-point kinds) or frame-of-reference offset, from the chunk's shared copy
template <int K, class T>
__device__ __forceinline__ T img_value(const uint64_t* tab, uint32_t x) {
  if (K == K_F64) return (T)__longlong_as_double((long long)tab[x]);
  if (K == K_F32) return (T)__int_as_float((int)(uint32_t)tab[x]);
  return (T)((int64_t)tab[0] + (int64_t)x);   // wraps to the element width exactly as the image builder verified
}
// consumer: registers <- stage (conflict-free: consecutive lanes read consecutive 16/8/4/2 bytes)
template <class PLAN, bool RT, int C>
__device__ __forceinline__ void load_col_staged(const RingArgs& a, const ColModes<PLAN>& cm, const uint64_t* imgsm, const uint8_t* stage, ColRegs<PLAN, C>& regs) {
  typedef typename KindT<PLAN::kind(C)>::T T;
  constexpr int K = PLAN::kind(C);
  const uint8_t* base = stage + stage_off<PLAN, RT, C>(a);
  regs.nullmask = 0;
  if (kind_has_image(K) && ((cm.img >> C) & 1)) {
    const uint64_t* tab = imgsm + img_col<PLAN, RT, C>(a);
    const bool w1 = (cm.w1 >> C) & 1;
#pragma unroll
    for (int u = 0; u < PLAN::RPT / 2; u++) {
      const int p = u * 2 * THREADS + 2 * (int)threadIdx.x;
      uint32_t x0, x1;
      if (w1) { const uint32_t x = *reinterpret_cast<const uint16_t*>(base + p); x0 = x & 0xffu; x1 = x >> 8; }
      else { const uint32_t x = *reinterpret_cast<const uint32_t*>(base + p * 2); x0 = x & 0xffffu; x1 = x >> 16; }
      regs.v[2 * u] = img_value<K, T>(tab, x0);
      regs.v[2 * u + 1] = img_value<K, T>(tab, x1);
    }
    return;
  }
#pragma unroll
  for (int u = 0; u < PLAN::RPT / 2; u++) {
    const int p = u * 2 * THREADS + 2 * (int)threadIdx.x;
    if (K == K_CODE) {
      if ((cm.c16 >> C) & 1) {
        uint32_t x = *reinterpret_cast<const uint32_t*>(base + p * 2);
        regs.v[2 * u] = (T)(int16_t)(x & 0xffffu);
        regs.v[2 * u + 1] = (T)(int16_t)(x >> 16);
      } else {
        int2 x = *reinterpret_cast<const int2*>(base + p * 4);
        regs.v[2 * u] = (T)x.x;
        regs.v[2 * u + 1] = (T)x.y;
      }
    } else if (sizeof(T) == 8) {
      longlong2 x = *reinterpret_cast<const longlong2*>(base + p * 8);
      regs.v[2 * u] = K == K_F64 ? (T)__longlong_as_double(x.x) : (T)x.x;
      regs.v[2 * u + 1] = K == K_F64 ? (T)__longlong_as_double(x.y) : (T)x.y;
    } else if (sizeof(T) == 4) {
      int2 x = *reinterpret_cast<const int2*>(base + p * 4);
      regs.v[2 * u] = K == K_F32 ? (T)__int_as_float(x.x) : (T)x.x;
      regs.v[2 * u + 1] = K == K_F32 ? (T)__int_as_float(x.y) : (T)x.y;
    } else if (sizeof(T) == 2) {
      uint32_t x = *reinterpret_cast<const uint32_t*>(base + p * 2);
      regs.v[2 * u] = (T)(int16_t)(x & 0xffffu);
      regs.v[2 * u + 1] = (T)(int16_t)(x >> 16);
    } else {
      uint16_t x = *reinterpret_cast<const uint16_t*>(base + p);
      regs.v[2 * u] = K == K_BOOL ? (T)((x & 0xff) == 1) : (T)(int8_t)(x & 0xff);
      regs.v[2 * u + 1] = K == K_BOOL ? (T)((x >> 8) == 1) : (T)(int8_t)(x >> 8);
    }
  }
}
// consumer, column with NULLs: row -> (is null, value index) through the null words; the value sits in the stage at
// [shift + (k - first) * w] where `first` is the tile's first stored value
template <class PLAN, bool RT, int C>
__device__ __forceinline__ void load_col_staged_nulls(const RingArgs& a, const DevCol& col, const ColModes<PLAN>& cm, int64_t tile_start, int num_rows,
                                                      const TileSmem<PLAN>& sm, const uint8_t* stage, ColRegs<PLAN, C>& regs) {
  typedef typename KindT<PLAN::kind(C)>::T T;
  constexpr int K = PLAN::kind(C);
  const int w = col_width<PLAN, C>(cm);   // (a column with NULLs in the batch has no image)
  const int n0 = col.tile_nulls[tile_start / NULL_PREFIX_ROWS];
  const int64_t first = tile_start - n0;
  const uint8_t* base = stage + stage_off<PLAN, RT, C>(a) + ((first * w) & 15);
  regs.nullmask = 0;
  // nulls before each 64-row word of the tile, computed BY EVERY WARP FOR ITSELF with shuffles (no shared memory, no CTA
  // barrier: warp-0-only preparation with two barriers per tile kept this path at a quarter of the roofline).  The rows of
  // a thread lie in word (u * THREADS / 32 + warp) for its row pair u, so a warp needs RPT / 2 of the tile's prefixes.
  constexpr int TW = TileSmem<PLAN>::TILE_WORDS;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int w0 = (int)(tile_start >> 6);
  uint64_t my_word = 0;
  if (lane < TW && w0 + lane < col.nwords) my_word = col.nulls[w0 + lane];
  int incl = __popcll(my_word);
  const int pc = incl;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += t; }
  const int excl = incl - pc;
#pragma unroll
  for (int r = 0; r < PLAN::RPT; r++) {
    const int li = row_in_tile(r);
    const int64_t i = tile_start + li;
    const int wi = (r >> 1) * (THREADS / 32) + warp;                      // == li >> 6
    const uint64_t word = __shfl_sync(0xffffffffu, my_word, wi);
    const int before = __shfl_sync(0xffffffffu, excl, wi);
    T v = (T)0;
    bool isnull = false;
    if (i < num_rows) {
      isnull = (word >> (i & 63)) & 1ull;
      const int64_t k = i - (n0 + before + __popcll(word & ((1ull << (i & 63)) - 1ull)));
      if (!isnull) {
        const uint8_t* p = base + (k - first) * w;
        if (K == K_CODE) v = (T)(w == 2 ? (int)*reinterpret_cast<const int16_t*>(p) : *reinterpret_cast<const int32_t*>(p));
        else if (K == K_BOOL) v = (T)(*p == 1);
        else v = *reinterpret_cast<const T*>(p);
      } else if (K == K_CODE) v = (T)col.dict_n;
    }
    regs.v[r] = v;
    regs.nullmask |= (isnull ? 1u : 0u) << r;
  }
}
template <class PLAN, bool RT, int C>
__device__ __forceinline__ void load_col_staged_any(const RingArgs& a, const DevCol& col, const ColModes<PLAN>& cm, const uint64_t* imgsm, int64_t tile_start, int num_rows,
                                                    const TileSmem<PLAN>& sm, const uint8_t* stage, ColRegs<PLAN, C>& regs) {
  if (PLAN::col_nullable(C) && col.nulls) load_col_staged_nulls<PLAN, RT, C>(a, col, cm, tile_start, num_rows, sm, stage, regs);
  else load_col_staged<PLAN, RT, C>(a, cm, imgsm, stage, regs);
}
template <class PLAN, bool RT, int... Cs>
__device__ __forceinline__ void load_all_staged_nulls(const RingArgs& a, const DevBatch<PLAN::NC>& b, const ColModes<PLAN>& cm, const uint64_t* imgsm, int64_t tile_start, const TileSmem<PLAN>& sm,
                                                      const uint8_t* stage, AllCols<PLAN, Seq<Cs...>>& regs, Seq<Cs...>) {
  int dummy[] = {0, (load_col_staged_any<PLAN, RT, Cs>(a, b.cols[Cs], cm, imgsm, tile_start, b.num_rows, sm, stage, static_cast<ColRegs<PLAN, Cs>&>(regs)), 0)...};
  (void)dummy;
}
template <class PLAN, bool RT, int... Cs>
__device__ __forceinline__ void load_all_staged(const RingArgs& a, const ColModes<PLAN>& cm, const uint64_t* imgsm, const uint8_t* stage, AllCols<PLAN, Seq<Cs...>>& regs, Seq<Cs...>) {
  int dummy[] = {0, (load_col_staged<PLAN, RT, Cs>(a, cm, imgsm, stage, static_cast<ColRegs<PLAN, Cs>&>(regs)), 0)...};
  (void)dummy;
}

// which batch a work item (chunk) belongs to: last b with chunk_prefix[b] <= item.  Items of a CTA increase
// monotonically, so `hint` (the previous answer) is advanced linearly before falling back to a binary search.
__device__ __forceinline__ int find_batch(const int32_t* chunk_prefix, int nbatches, int item, int hint) {
  if (hint >= 0) {
    int b = hint;
#pragma unroll 1
    for (int step = 0; step < 4 && b + 1 < nbatches && chunk_prefix[b + 1] <= item; step++) b++;
    if (b + 1 >= nbatches || chunk_prefix[b + 1] > item) return b;
  }
  int lo = 0, hi = nbatches;
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (chunk_prefix[mid] <= item) lo = mid; else hi = mid;
  }
  return lo;
}

// context handed to the generated row functions
struct RowCtx {
  const Literals* L;
  const int32_t* radix;
  // per-batch tables of this plan, refreshed once per chunk:
  //   aux = [int32 offset x NT][pad to 8][uint64 kpack x NT][tables...]
  //   tbl[t]   : table t (truth table: uint8 per dictionary code; key map: int32 group id per code)
  //   kpack[t] : key maps of <= 8 codes packed one byte per code (no memory access per row), else ~0
  const uint8_t* tbl[MAX_TABLES];
  uint64_t kpack[MAX_TABLES];
  const uint8_t* litpool;           // STRING literal bytes of this execution
  const uint8_t* strbase[64];       // per STRING scan column: body of an ENC_STR_RAW batch (refs are positions into it), else nullptr
  uint64_t ord;                     // plans with FIRST / LAST: the current row's order key without its NULL flag
  __device__ __forceinline__ const uint8_t* table(int t) const { return tbl[t]; }
  __device__ __forceinline__ const uint8_t* lit_bytes(int slot) const { return litpool + (uint32_t)((uint64_t)L->i[slot] >> 32); }
  __device__ __forceinline__ int lit_len(int slot) const { return (int)((uint64_t)L->i[slot] & 0xffffffffull); }
  // record of a STRING value held by reference: raw batch -> body + position; dictionary batch -> entry address from the
  // per-batch key-pointer table t (int64 per code)
  __device__ __forceinline__ int64_t str_ref(int c, int t, int code) const {
    return strbase[c] ? (int64_t)(uintptr_t)(strbase[c] + (uint32_t)code) : reinterpret_cast<const int64_t*>(tbl[t])[code];
  }
  __device__ __forceinline__ int key_id(int t, int code) const {
    const uint64_t kp = kpack[t];
    return kp != ~0ull ? (int)((kp >> (code * 8)) & 0xffull) : reinterpret_cast<const int32_t*>(tbl[t])[code];
  }
};
template <int NT>
__device__ __forceinline__ void load_tables(RowCtx& ctx, const uint8_t* aux) {
  if (NT > 0) {
    const int32_t* off = reinterpret_cast<const int32_t*>(aux);
    const uint64_t* kp = reinterpret_cast<const uint64_t*>(aux + ((4 * NT + 7) & ~7));
#pragma unroll
    for (int t = 0; t < NT; t++) { ctx.tbl[t] = aux + __ldg(&off[t]); ctx.kpack[t] = __ldg(&kp[t]); }
  }
}

// per chunk: which STRING columns of this batch are raw (ENC_STR_RAW)
template <class PLAN, int... Cs>
__device__ __forceinline__ void load_strbase(RowCtx& ctx, const DevBatch<PLAN::NC>& b, Seq<Cs...>) {
  int dummy[] = {0, (PLAN::kind(Cs) == K_CODE ? (ctx.strbase[Cs] = (b.cols[Cs].enc == ENC_STR_RAW ? b.cols[Cs].dict : nullptr), 0) : 0)...};
  (void)dummy;
}

// what the staged loads of batch b read (images only when the launch has room for their tables: with_img; never in the
// variant with the per-row paths, whose register budget they would take)
template <class PLAN, int... Cs>
__device__ __forceinline__ ColModes<PLAN> col_modes(const DevBatch<PLAN::NC>& b, bool with_img, Seq<Cs...>) {
  typedef SD_CMASK(PLAN) M;
  ColModes<PLAN> cm;
  cm.c16 = 0; cm.img = 0; cm.w1 = 0;
  int dummy[] = {0, (PLAN::kind(Cs) == K_CODE ? (cm.c16 |= (M)(b.cols[Cs].enc == ENC_DICTIONARY ? 1 : 0) << Cs, 0) : 0)...};
  if (PLAN::STAGES > 0 && !PLAN::SLOW_PATHS && with_img) {
    int d1[] = {0, (kind_has_image(PLAN::kind(Cs)) && b.cols[Cs].img
                    ? (cm.img |= (M)1 << Cs, cm.w1 |= (M)(b.cols[Cs].img_w == 1) << Cs, 0) : 0)...};
    (void)d1;
  }
  (void)dummy;
  return cm;
}
// the chunk's img_tab words -> shared memory (the caller brackets this with consumer barriers)
template <class PLAN, bool RT, int... Cs>
__device__ __forceinline__ void load_img_tables(const RingArgs& a, const DevBatch<PLAN::NC>& b, const ColModes<PLAN>& cm, uint64_t* imgsm, Seq<Cs...>) {
  int dummy[] = {0, (kind_has_image(PLAN::kind(Cs)) && ((cm.img >> Cs) & 1)
                     ? ([&] { for (int i = threadIdx.x; i < b.cols[Cs].img_n; i += THREADS) imgsm[img_col<PLAN, RT, Cs>(a) + i] = __ldg(&b.cols[Cs].img_tab[i]); }(), 0) : 0)...};
  (void)dummy;
}

// ================================================================================================
// The kernel.  dynamic shared memory: [TileSmem<PLAN>] [private group tables | reduction scratch]
// ================================================================================================
// (the body of both kernels below; RT: the ring layout of the launch, `rl`, instead of the verbatim one)
template <class PLAN, bool RT>
__device__ __forceinline__ void scan_aggregate(const ScanArgs args, const RingArgs rl) {
  typedef typename MakeSeq<PLAN::NC>::type ColSeq;
  constexpr int NSLOT = PLAN::NSLOT;
  constexpr int RPT = PLAN::RPT;
  constexpr int TILE_ROWS = THREADS * RPT;
  const int CHUNK_TILES = args.chunk_rows / TILE_ROWS;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  TileSmem<PLAN>& sm = *reinterpret_cast<TileSmem<PLAN>*>(smem_raw);
  uint64_t* table = reinterpret_cast<uint64_t*>(smem_raw + ((sizeof(TileSmem<PLAN>) + 15) & ~size_t(15)));
  const int tid = threadIdx.x;
  const int NE = args.ngroups * NSLOT;   // entries of the group table
  const DevBatch<PLAN::NC>* batches = reinterpret_cast<const DevBatch<PLAN::NC>*>(args.batches);

  // ---- staged fast path: [full barriers][empty barriers][ring of nstages stages] -----------------------
  // The ring starts on a 128-byte boundary of the shared window, so that every bulk copy lands 128-byte aligned (each
  // column region of a stage is a multiple of 128 bytes).  Dynamic shared memory itself starts behind the kernel's static
  // shared variables, at an address that is only 16-byte aligned: the engine reserves RING_ALIGN_SLACK bytes for this.
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_raw + args.ring_off);
  uint64_t* empty_bar = full_bar + MAX_STAGES;
  uint8_t* ring = smem_raw + ((smem_u32(smem_raw) + args.ring_off + 2 * MAX_STAGES * 8 + 127) & ~127u) - smem_u32(smem_raw);
  const int nstages = args.nstages;
  if (PLAN::STAGES > 0) {
    if (tid == 0) {
      for (int i = 0; i < nstages; i++) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], THREADS / 32); }

      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();   // all THREADS + 32 threads: the only CTA-wide barrier the producer warp joins
    if (tid >= THREADS) {
      // ---- producer warp: one lane walks the same work sequence and keeps the ring full -----------
      if (tid == THREADS) {
        int stage = 0;
        uint32_t phase = 0;
        int p_hint = -1;
        for (int item = blockIdx.x; item < args.total_chunks; item += gridDim.x) {
          const int bi = find_batch(args.chunk_prefix, args.nbatches, item, p_hint);
          p_hint = bi;
          const DevBatch<PLAN::NC>& b = batches[bi];
          if (!(b.flags & (BATCH_ALL_FAST | (PLAN::SLOW_PATHS ? BATCH_FAST_OVERLAY : 0) | (PLAN::ANY_NULLABLE ? BATCH_FAST_NULLS : 0)))) continue;
          const int chunk = item - args.chunk_prefix[bi];
          const int num_rows = b.num_rows;
          const int ntiles = (num_rows + TILE_ROWS - 1) / TILE_ROWS;
          const int tile0 = chunk * CHUNK_TILES, tile_end = min(tile0 + CHUNK_TILES, ntiles);
          const ColModes<PLAN> cm = col_modes<PLAN>(b, args.img_off >= 0, ColSeq());
          ProducerCols<PLAN::NC> pc;
          load_producer_cols<PLAN>(b, cm, pc, ColSeq());
          for (int tile = tile0; tile < tile_end; tile++) {
            const int64_t tile_start = (int64_t)tile * TILE_ROWS;
            const int rows = min(TILE_ROWS, num_rows - (int)tile_start);
            mbar_wait(&empty_bar[stage], phase ^ 1u);
            issue_tile_copies<PLAN, RT>(rl, pc, cm, tile_start, rows, ring + (size_t)stage * stage_size<PLAN, RT>(rl), &full_bar[stage], ColSeq());
            if (++stage == nstages) { stage = 0; phase ^= 1u; }
          }
        }
      }
      return;
    }
  }
  int c_stage = 0;
  uint32_t c_phase = 0;
  int c_hint = -1;
  // per-chunk shared copies of the image tables (at args.img_off); refreshed when a work item's batch differs from the
  // last one loaded
  int img_batch = -1;

  // ---- accumulator init -------------------------------------------------------------------------
  uint64_t acc[NSLOT > 0 ? NSLOT : 1];
  constexpr int RG = PLAN::MODE == MODE_GROUPS ? PLAN::REG_GROUPS : 0;   // > 0: group table in registers
  uint64_t racc[RG > 0 ? RG : 1][NSLOT > 0 ? NSLOT : 1];
  if (RG > 0) {
#pragma unroll
    for (int gi = 0; gi < RG; gi++)
#pragma unroll
      for (int s = 0; s < NSLOT; s++) racc[gi][s] = slot_identity(PLAN::slot_op(s));
  } else if (PLAN::MODE == MODE_NOKEY) {
#pragma unroll
    for (int s = 0; s < NSLOT; s++) acc[s] = slot_init<PLAN>(PLAN::slot_op(s));
  } else if (PLAN::MODE == MODE_HASH || PLAN::MODE == MODE_PROJECT || PLAN::MODE == MODE_MUTATE) {
    // nothing per CTA: the table / output buffer is global
  } else if (args.table_mode == TABLE_PRIVATE) {
    // private table of thread t: entry e at table[e * THREADS + t]: lanes hit distinct banks
    for (int e = 0; e < NE; e++) table[e * THREADS + tid] = slot_init<PLAN>(PLAN::slot_op(e % NSLOT));
  } else if (args.table_mode == TABLE_SHARED_ATOMIC) {
    for (int e = tid; e < NE; e += THREADS) table[e] = slot_init<PLAN>(PLAN::slot_op_rt(e % NSLOT));
    consumer_sync();
  }
  // moment aggregates: where a row finds its group's K (sd_device.h SHIFT_EMPTY).  The words beside the running result / hash
  // entries hold it; no-key plans keep it in registers once read, private / shared-atomic dense tables a per-CTA copy in shared
  // memory they fill on first touch
  constexpr int NSH = PlanShifts<PLAN>::N;
  static_assert(NSH == 0 || RG == 0, "the register-table variant is never built for plans with moment aggregates");
  constexpr int NORD = PlanOrders<PLAN>::N;
  static_assert(NORD == 0 || RG == 0, "the register-table variant is never built for plans with FIRST / LAST");
  uint64_t kreg[NSH > 0 ? NSH : 1];
  uint64_t* kcache = nullptr;
  (void)kreg; (void)kcache;
  if constexpr (NSH > 0) {
#pragma unroll
    for (int i = 0; i < NSH; i++) kreg[i] = SHIFT_EMPTY;
    if (PLAN::MODE == MODE_GROUPS && args.shift_cache_off >= 0) {
      kcache = reinterpret_cast<uint64_t*>(smem_raw + args.shift_cache_off);
      for (int e = tid; e < args.ngroups * NSH; e += THREADS) kcache[e] = SHIFT_EMPTY;
      consumer_sync();
    }
  }
  unsigned long long n_scanned = 0, n_passed = 0;   // flushed from 32-bit per-chunk counters
#if SD_EXP_SKIP_ROWS || SD_EXP_SINK_GROUPS
  uint64_t exp_sink = 0;
  uint64_t exp_acc[NSLOT > 0 ? NSLOT : 1];
#pragma unroll
  for (int s = 0; s < NSLOT; s++) exp_acc[s] = 0;
#endif

  RowCtx ctx;
  ctx.L = &args.lits;
  ctx.radix = args.radix;
  ctx.litpool = args.lit_pool;

  // ---- persistent loop over (batch, chunk) work items, static round-robin -------------------------
  for (int item = blockIdx.x; item < args.total_chunks; item += gridDim.x) {
    const int lo = find_batch(args.chunk_prefix, args.nbatches, item, c_hint);
    c_hint = lo;
    const DevBatch<PLAN::NC>& b = batches[lo];
    const int chunk = item - args.chunk_prefix[lo];
    const int num_rows = b.num_rows;
    const bool overlay = PLAN::SLOW_PATHS && (b.flags & BATCH_FAST_OVERLAY) != 0;
    const bool with_nulls = PLAN::ANY_NULLABLE && (b.flags & BATCH_FAST_NULLS) != 0 && PLAN::STAGES > 0;
    const bool fast = (b.flags & BATCH_ALL_FAST) != 0 || ((overlay || with_nulls) && PLAN::STAGES > 0);
    // the staged-only variant of a plan (SLOW_PATHS == false) is launched on batches of the staged kinds only; anything
    // else reaching it is a host-side bug: stop loudly instead of aggregating garbage
    if (!PLAN::SLOW_PATHS && !fast) __trap();
    load_tables<PLAN::NTABLES>(ctx, b.aux);
    if (PLAN::ANY_STRING) load_strbase<PLAN>(ctx, b, ColSeq());
    const ColModes<PLAN> cm = col_modes<PLAN>(b, args.img_off >= 0, ColSeq());
    if (PLAN::STAGES > 0 && !PLAN::SLOW_PATHS && fast && cm.img && lo != img_batch) {
      consumer_sync();   // every consumer is done with the previous batch's tables
      load_img_tables<PLAN, RT>(rl, b, cm, reinterpret_cast<uint64_t*>(smem_raw + args.img_off), ColSeq());
      consumer_sync();
      img_batch = lo;
    }
    uint32_t c_scanned = 0, c_passed = 0;
    const int tile0 = chunk * CHUNK_TILES;
    const int ntiles = (num_rows + TILE_ROWS - 1) / TILE_ROWS;
    const int tile_end = min(tile0 + CHUNK_TILES, ntiles);

    for (int tile = tile0; tile < tile_end; tile++) {
      const int64_t tile_start = (int64_t)tile * TILE_ROWS;
      AllCols<PLAN, ColSeq> regs;
      uint32_t live = 0;   // bit r: row exists and is not deleted
#pragma unroll
      for (int r = 0; r < RPT; r++) live |= (tile_start + row_in_tile(r) < num_rows ? 1u : 0u) << r;

      if (fast) {
        if (PLAN::STAGES > 0) {
          mbar_wait(&full_bar[c_stage], c_phase);   // (the NULL-aware loads derive their word prefixes per warp: no barrier here)
          const uint64_t* imgsm = reinterpret_cast<const uint64_t*>(smem_raw + args.img_off);   // (read only where cm.img)
          if (with_nulls) load_all_staged_nulls<PLAN, RT>(rl, b, cm, imgsm, tile_start, sm, ring + (size_t)c_stage * stage_size<PLAN, RT>(rl), regs, ColSeq());
          else load_all_staged<PLAN, RT>(rl, cm, imgsm, ring + (size_t)c_stage * stage_size<PLAN, RT>(rl), regs, ColSeq());
          // The rows of this tile are in registers now: release the stage.  The stage was read through the GENERIC proxy (ld.shared)
          // and will be refilled through the ASYNC proxy (cp.async.bulk): the mbarrier alone does not order the two (PTX ISA, "async
          // proxy": accesses to the same location across proxies need a cross-proxy fence).  Without the fence a refill can land
          // while loads issued before the release are still pending -- seen when the LSU is busy with a hash plan's global
          // atomics: ~1 % of the staged values then belong to the stage's NEXT tile.
#ifndef SD_EXP_NO_PROXY_FENCE   // (diagnostic builds reproduce the failure with -DSD_EXP_NO_PROXY_FENCE)
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
#endif
          __syncwarp();
          if ((tid & 31) == 0) mbar_arrive(&empty_bar[c_stage]);
#if SD_EXP_VERIFY
          if (!with_nulls) {
            AllCols<PLAN, ColSeq> chk;
            load_all_fast<PLAN>(b, tile_start, chk, ColSeq());
            verify_all<PLAN>(regs, chk, live, tile_start, c_stage, args.counters, b, nstages, PLAN::MODE == MODE_HASH ? args.hash.overflow : nullptr, ColSeq());
          }
#endif
          if (++c_stage == nstages) { c_stage = 0; c_phase ^= 1u; }
        } else {
          load_all_fast<PLAN>(b, tile_start, regs, ColSeq());
        }
      }
      if (PLAN::SLOW_PATHS && fast && overlay) {
        // staged tile + update deltas / delete mask: every warp patches its own rows from its own cursors (no CTA barrier)
        warp_overlay_all<PLAN>(b, tile_start, tile == tile0, sm, regs, live, ColSeq());
      } else if (PLAN::SLOW_PATHS && !fast) {
        // per-row decode of the whole tile; drops the deleted rows
        consumer_sync();                       // previous tile's readers are done with sm
        clear_upd_bits<PLAN>(b, sm, ColSeq());
        if (tid < 32) find_all_ranges<PLAN>(b, tile_start, tile == tile0, sm, tid, ColSeq());
        consumer_sync();
        prep_all_general<PLAN>(b, tile_start, sm, ColSeq());
        if (b.deletes) {                       // delete mask -> tile bitmap (enc/ColumnDeleteDecoder.scala:49-55)
          const int32_t ts = (int32_t)tile_start;
          for (int j = sm.delrange[0] + tid; j < sm.delrange[1]; j += THREADS) {
            const int li = b.deletes[j] - ts;
            atomicOr(&sm.delbits[li >> 5], 1u << (li & 31));
          }
        }
        consumer_sync();
        load_all_general<PLAN>(b, tile, tile_start, sm, regs, ColSeq());
        if (b.deletes) {
#pragma unroll
          for (int r = 0; r < RPT; r++) {
            const int li = row_in_tile(r);
            if ((sm.delbits[li >> 5] >> (li & 31)) & 1u) live &= ~(1u << r);
          }
        }
      }

      // ---- row at a time over registers: filter -> group -> accumulate -------------------------
      c_scanned += __popc(live);
#if SD_EXP_SKIP_ROWS
      fold_all<PLAN>(regs, exp_sink, ColSeq());
      continue;
#endif
      if (PLAN::MODE == MODE_PROJECT || PLAN::MODE == MODE_MUTATE) {
        // filter -> project: passing rows become fixed-width records; one atomic per warp per row slot
        constexpr int NP = PLAN::NPROJ > 0 ? PLAN::NPROJ : 1;
        constexpr int HDR = PLAN::MODE == MODE_MUTATE ? 2 : 1;   // MODE_MUTATE: (batch, row) key word + null word
        constexpr int REC = 8 * HDR + 8 * NP;
#pragma unroll
        for (int r = 0; r < RPT; r++) {
          bool pass = false;
          uint64_t pv[NP];
          uint32_t pnull = 0;
          if ((live >> r) & 1u) {
            typename PLAN::Row row;
            fill_row<PLAN>(regs, r, row, ColSeq());
            pass = PLAN::filter(row, ctx);
            if (pass) PLAN::project(row, ctx, pv, pnull);
          }
          const unsigned m = __ballot_sync(0xffffffffu, pass);
          if (m) {
            const int lane_id = tid & 31, leader = __ffs(m) - 1;
            unsigned long long base = 0;
            if (lane_id == leader) base = atomicAdd(args.out_count, (unsigned long long)__popc(m));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (pass) {
              c_passed++;
              const unsigned long long idx = base + __popc(m & ((1u << lane_id) - 1u));
              if ((int64_t)idx < args.out_cap) {
                uint64_t* rec = reinterpret_cast<uint64_t*>(args.out_rows + idx * REC);
                if (PLAN::MODE == MODE_MUTATE) {
                  rec[0] = ((uint64_t)(uint32_t)(args.batch_base + lo) << 32) | (uint32_t)(tile_start + row_in_tile(r));
                  rec[1] = pnull;
                } else {
                  rec[0] = (uint64_t)(uint32_t)(args.batch_base + lo) | ((uint64_t)pnull << 32);
                }
#pragma unroll
                for (int j = 0; j < PLAN::NPROJ; j++) rec[HDR + j] = pv[j];
              }
            }
          }
        }
        continue;
      }
#pragma unroll
      for (int r = 0; r < RPT; r++) {
        if (!((live >> r) & 1u)) continue;
        typename PLAN::Row row;
        fill_row<PLAN>(regs, r, row, ColSeq());
        if (!PLAN::filter(row, ctx)) continue;      // FilterExec: only TRUE passes
        c_passed++;
        uint64_t sv[NSLOT > 0 ? NSLOT : 1];
        if constexpr (NORD > 0)   // the row's order key (sd_device.h ORDER_EMPTY_FIRST) without its NULL flag
          ctx.ord = ((uint64_t)(uint32_t)(args.batch_base + lo + 1) << 32) | ((uint64_t)(uint32_t)(tile_start + row_in_tile(r)) << 1);
        PLAN::slots(row, ctx, sv);
        if (PLAN::MODE == MODE_NOKEY) {
          if constexpr (NSH > 0)
            apply_shifts<PLAN>(sv, [&](int i, uint64_t c) {
              if (kreg[i] == SHIFT_EMPTY) kreg[i] = shift_claim(args.shifts + i, c);
              return kreg[i];
            });
          if constexpr (NORD > 0) combine_plain<PLAN>(acc, 1, sv);
          else {
#pragma unroll
            for (int s = 0; s < NSLOT; s++) acc[s] = slot_combine(PLAN::slot_op(s), acc[s], sv[s]);
          }
        } else {
          if (PLAN::MODE == MODE_HASH) {
            int64_t kc[PLAN::NKEYS > 0 ? PLAN::NKEYS : 1];
            uint32_t knull = 0;
            PLAN::keys(row, ctx, kc, knull);
            const int64_t e = hash_find_or_insert<(PLAN::NKEYS > 0 ? PLAN::NKEYS : 1), PLAN::STRKEYMASK>(args.hash, kc, knull);
            if (e >= 0) {
              uint64_t* t = args.hash.vals + (size_t)e * NSLOT;
              if constexpr (NSH > 0) apply_shifts<PLAN>(sv, [&](int i, uint64_t c) { return shift_claim(args.hash.shifts + (size_t)e * NSH + i, c); });
              if constexpr (NORD > 0) combine_atomic<PLAN, false>(t, sv);
              else {
#pragma unroll
                for (int s = 0; s < NSLOT; s++) slot_atomic(PLAN::slot_op(s), t + s, sv[s]);
              }
            }
            continue;
          }
          const int g = PLAN::group(row, ctx);
          if constexpr (NSH > 0) {
            uint64_t* kg = args.shifts + (size_t)g * NSH;
            if (kcache)
              apply_shifts<PLAN>(sv, [&](int i, uint64_t c) {
                uint64_t k = kcache[g * NSH + i];
                if (k == SHIFT_EMPTY) { k = shift_claim(kg + i, c); kcache[g * NSH + i] = k; }
                return k;
              });
            else
              apply_shifts<PLAN>(sv, [&](int i, uint64_t c) { return shift_claim(kg + i, c); });
          }
          if (RG > 0) {   // predicated register accumulators: no memory traffic, no dependent smem chains
#pragma unroll
            for (int gi = 0; gi < RG; gi++) {
              if (g == gi) {
#pragma unroll
                for (int s = 0; s < NSLOT; s++) racc[gi][s] = slot_combine(PLAN::slot_op(s), racc[gi][s], sv[s]);
              }
            }
          } else if (args.table_mode == TABLE_PRIVATE) {
#if SD_EXP_SINK_GROUPS   // (diagnostic builds: the slots and the group are computed, the table is never touched)
            exp_sink += (uint64_t)g;
            if constexpr (NORD > 0) combine_plain<PLAN>(exp_acc, 1, sv);
            else {
#pragma unroll
              for (int s = 0; s < NSLOT; s++) exp_acc[s] = slot_combine(PLAN::slot_op(s), exp_acc[s], sv[s]);
            }
            continue;
#endif
            uint64_t* t = table + (size_t)g * NSLOT * THREADS + tid;
            if constexpr (NORD > 0) combine_plain<PLAN>(t, THREADS, sv);
            else {
#pragma unroll
              for (int s = 0; s < NSLOT; s++) t[s * THREADS] = slot_combine(PLAN::slot_op(s), t[s * THREADS], sv[s]);
            }
          } else if constexpr (NORD > 0) {
            if (args.table_mode == TABLE_SHARED_ATOMIC) combine_atomic<PLAN, true>(table + (size_t)g * NSLOT, sv);
            else combine_atomic<PLAN, false>(args.result + (size_t)g * NSLOT, sv);
          } else {
            uint64_t* t = (args.table_mode == TABLE_SHARED_ATOMIC ? table : args.result) + (size_t)g * NSLOT;
#pragma unroll
            for (int s = 0; s < NSLOT; s++) slot_atomic(PLAN::slot_op(s), t + s, sv[s]);
          }
        }
      }
    }
    n_scanned += c_scanned;
    n_passed += c_passed;
  }

  // ---- CTA reduction (fixed order) -> partials[blockIdx] -------------------------------------------
  consumer_sync();
  uint64_t* my_partials = args.partials + (size_t)blockIdx.x * NE;
  const int lane = tid & 31, warp = tid >> 5;
  if (PLAN::MODE == MODE_HASH || PLAN::MODE == MODE_PROJECT || PLAN::MODE == MODE_MUTATE) {
    // results live in the global hash table / the output record buffer
  } else if (PLAN::MODE == MODE_NOKEY) {
    uint64_t* scratch = table;   // [NSLOT][THREADS/32]
#pragma unroll
    for (int s = 0; s < NSLOT; s++) {
      if constexpr (NORD > 0) {
        const int op = PLAN::slot_op(s);
        if (op == SLOT_PAIR_VAL) continue;
        if (is_order_op(op)) {
          uint64_t k = acc[s], v = acc[s + 1];
#pragma unroll
          for (int d = 16; d > 0; d >>= 1) order_combine(op, k, v, __shfl_xor_sync(0xffffffffu, k, d), __shfl_xor_sync(0xffffffffu, v, d));
          if (lane == 0) { scratch[s * (THREADS / 32) + warp] = k; scratch[(s + 1) * (THREADS / 32) + warp] = v; }
          continue;
        }
      }
      uint64_t v = acc[s];
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) v = slot_combine(PLAN::slot_op(s), v, __shfl_xor_sync(0xffffffffu, v, d));
      if (lane == 0) scratch[s * (THREADS / 32) + warp] = v;
    }
    consumer_sync();
    if (NORD > 0 && tid < NSLOT && is_order_op(PLAN::slot_op_rt(tid))) {
      const int op = PLAN::slot_op_rt(tid);
      uint64_t k = slot_initial(op), v = 0;
      for (int w = 0; w < THREADS / 32; w++) order_combine(op, k, v, scratch[tid * (THREADS / 32) + w], scratch[(tid + 1) * (THREADS / 32) + w]);
      my_partials[tid] = k;
      my_partials[tid + 1] = v;
    } else if (NORD > 0 && tid < NSLOT && PLAN::slot_op_rt(tid) == SLOT_PAIR_VAL) {
      // written with its key
    } else if (tid < NSLOT) {
      const int op = PLAN::slot_op_rt(tid);
      uint64_t v = slot_identity(op);
      for (int w = 0; w < THREADS / 32; w++) v = slot_combine(op, v, scratch[tid * (THREADS / 32) + w]);
      my_partials[tid] = v;
    }
  } else if (args.table_mode == TABLE_SHARED_ATOMIC) {
    for (int e = tid; e < NE; e += THREADS) my_partials[e] = table[e];
  } else if (args.table_mode == TABLE_PRIVATE || RG > 0) {
    if (RG > 0) {   // spill the register tables into the (now idle) ring in the private-table layout
      table = reinterpret_cast<uint64_t*>(ring);
#pragma unroll
      for (int gi = 0; gi < RG; gi++)
        if (gi < args.ngroups) {
#pragma unroll
          for (int s = 0; s < NSLOT; s++) table[(gi * NSLOT + s) * THREADS + tid] = racc[gi][s];
        }
      consumer_sync();
    }
    for (int e = warp; e < NE; e += THREADS / 32) {
      const int op = PLAN::slot_op_rt(e % NSLOT);
      if constexpr (NORD > 0) {
        if (op == SLOT_PAIR_VAL) continue;
        if (is_order_op(op)) {
          uint64_t k = slot_initial(op), v = 0;
#pragma unroll
          for (int j = 0; j < THREADS / 32; j++) order_combine(op, k, v, table[e * THREADS + lane + 32 * j], table[(e + 1) * THREADS + lane + 32 * j]);
#pragma unroll
          for (int d = 16; d > 0; d >>= 1) order_combine(op, k, v, __shfl_xor_sync(0xffffffffu, k, d), __shfl_xor_sync(0xffffffffu, v, d));
          if (lane == 0) { my_partials[e] = k; my_partials[e + 1] = v; }
          continue;
        }
      }
      uint64_t v = slot_identity(op);
#pragma unroll
      for (int j = 0; j < THREADS / 32; j++) v = slot_combine(op, v, table[e * THREADS + lane + 32 * j]);
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) v = slot_combine(op, v, __shfl_xor_sync(0xffffffffu, v, d));
      if (lane == 0) my_partials[e] = v;
    }
  }
#if SD_EXP_SKIP_ROWS || SD_EXP_SINK_GROUPS
  {   // the sinks feed a store that (almost) never happens, so the work that fills them survives
#pragma unroll
    for (int s = 0; s < NSLOT; s++) exp_sink ^= exp_acc[s];
    if (exp_sink == 0x5d5d5d5d5d5d5d5dull) args.counters[7] = exp_sink;
  }
#endif
  // metrics
  {
    unsigned long long a = n_scanned, p = n_passed;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, d); p += __shfl_xor_sync(0xffffffffu, p, d); }
    if (lane == 0) { atomicAdd(&args.counters[0], a); atomicAdd(&args.counters[1], p); }
  }

  // ---- last CTA combines all CTA partials in CTA order into the running result ---------------------
  __shared__ bool is_last;
  __threadfence();
  consumer_sync();
  if (tid == 0) is_last = atomicAdd(args.ticket, 1u) == gridDim.x - 1;
  consumer_sync();
  if (is_last && PLAN::MODE != MODE_HASH && PLAN::MODE != MODE_PROJECT && PLAN::MODE != MODE_MUTATE && !(PLAN::MODE == MODE_GROUPS && args.table_mode == TABLE_GLOBAL_ATOMIC)) {
    __threadfence();
    for (int e = tid; e < NE; e += THREADS) {
      const int op = PLAN::slot_op_rt(e % NSLOT);
      if constexpr (NORD > 0) {
        if (op == SLOT_PAIR_VAL) continue;
        if (is_order_op(op)) {
          uint64_t k = slot_initial(op), v = 0;
          for (unsigned bk = 0; bk < gridDim.x; bk++)
            order_combine(op, k, v, __ldcg(&args.partials[(size_t)bk * NE + e]), __ldcg(&args.partials[(size_t)bk * NE + e + 1]));
          if (!args.fresh) { uint64_t rk = args.result[e], rv = args.result[e + 1]; order_combine(op, rk, rv, k, v); k = rk; v = rv; }
          args.result[e] = k;
          args.result[e + 1] = v;
          continue;
        }
      }
      uint64_t v = slot_identity(op);
      for (unsigned bk = 0; bk < gridDim.x; bk++) v = slot_combine(op, v, __ldcg(&args.partials[(size_t)bk * NE + e]));
      args.result[e] = args.fresh ? v : slot_combine(op, args.result[e], v);
    }
  }
  if (is_last && tid == 0) *args.ticket = 0;
}

template <class PLAN>
__global__ void __launch_bounds__(THREADS + (PLAN::STAGES > 0 ? 32 : 0), PLAN::MIN_CTAS) scan_aggregate_kernel(const ScanArgs args) {
  scan_aggregate<PLAN, false>(args, RingArgs{});
}

// A dense group-by's staged-only variant also has a kernel for two CTAs per SM, launched when the launch's compact ring
// (RingArgs), the private table and the image tables fit half the SM (sd_engine.cu launch_scan): 2 x 9 warps on the SM's
// four register partitions need <= 96 registers per thread, a cap the one-CTA kernel must not pay (wide plans would spill).
template <class PLAN>
struct TwoCtaKernel {
  static constexpr bool BUILT = PLAN::MODE == MODE_GROUPS && !PLAN::SLOW_PATHS && PLAN::STAGES > 0 && PLAN::REG_GROUPS == 0;
};
template <class PLAN>
__global__ void __launch_bounds__(THREADS + 32, 2) scan_aggregate_kernel_2cta(const ScanArgs args, const RingArgs ring) {
  scan_aggregate<PLAN, true>(args, ring);
}
#ifndef __CUDACC_RTC__
// the two-CTA kernel of PLAN for the registry, or nullptr
template <class PLAN>
const void* two_cta_kernel() {
  if constexpr (TwoCtaKernel<PLAN>::BUILT) return (const void*)&scan_aggregate_kernel_2cta<PLAN>;
  else return nullptr;
}
#endif

}  // namespace sd
#endif
