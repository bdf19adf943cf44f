// sd_encode.cu -- ColumnBatch creation on the device (SURVEY.md 8f N2): raw column values of an ingest batch -> the
// reference's encoded column buffers + stats row, resident in an sd_store, without a host round trip of the values.
//
// Restates, as whole-column kernels, what the reference does row by row in its generated insert loop:
//   ColumnInsertExec.doProduce / ColumnWriter         core/execution/columnar/ColumnInsertExec.scala:326-822, 848-921
//   ColumnEncoder.initialize / writeIsNull / finish   enc/ColumnEncoding.scala:177-736, 1145-1332 (null words, trimmed)
//   UncompressedEncoder                               enc/Uncompressed.scala:228-448
//   DictionaryEncoder (first-seen order, int16 -> int32 indexes at 32767 entries)   enc/DictionaryEncoding.scala:168-450
//   BooleanBitSetEncoder                              enc/BooleanBitSetEncoding.scala:62-152
//   default encoder choice                            enc/ColumnEncoding.scala:837-844  (STRING -> Dictionary, BOOLEAN -> BitSet,
//                                                     everything else Uncompressed)
// The byte layout is the one snappydata_b200/column_format.py writes (the fixture writer stays the spec): the tests decode
// device-encoded batches with the oracle and compare them byte for byte with the fixture writer's output.
//
// Work split: the device does everything that touches every row (null words, compaction of the non-null values, the boolean
// bit set, finding the distinct strings and their first occurrence, rewriting strings as dictionary indexes, min / max);
// the host only lays out the buffer (header, trimmed null words, the dictionary in first-seen order) from a few KB of
// feedback.  The phases after the raw values are on the device (enc_null_words_many / enc_queue_words / enc_first_seen_dict / enc_layout / enc_write, declared in
// sd_host.h) are shared with compaction (sd_compact.cu), which feeds them the materialised columns of many batches at once.
#include <algorithm>
#include <climits>
#include <cstring>
#include <functional>

#include "sd_host.h"

namespace sd {

// shared with sd_store.cu: registers a column whose header / null words / dictionary ("prefix") the host knows and whose
// body a kernel writes at the returned device address
int store_register_encoded(sd_store* s, const uint8_t* prefix, int64_t prefix_len, int64_t total_len, int type, int nullable,
                           int num_rows, StoredCol& c);

namespace {

enum : int32_t { EK_I8 = 0, EK_I16, EK_I32, EK_I64, EK_F32, EK_F64, EK_BOOL, EK_STRCODE16, EK_STRCODE32 };

struct EncCol {
  const uint8_t* values;     // raw values, one per row (EK_STRCODE*: int32 slot per row)
  const uint8_t* nulls;      // 1 byte per row or nullptr
  const int32_t* slot_code;  // EK_STRCODE*: dictionary code per hash slot
  uint8_t* out;              // body: compacted values / bit-set words / dictionary indexes
  uint64_t* stat;            // [0] lower, [1] upper (raw bits of the value type), [2] non-null count
  int32_t kind;
  int32_t n;
};

__device__ __forceinline__ void null_word(const uint8_t* nulls, int n, uint64_t* words, int* fb, int w) {
  if ((int64_t)w * 64 >= n) return;
  uint64_t word = 0;
  const int lim = min(64, n - w * 64);
  for (int b = 0; b < lim; b++) word |= (uint64_t)(nulls[(int64_t)w * 64 + b] != 0) << b;
  words[w] = word;
  if (word) { atomicAdd(&fb[0], __popcll(word)); atomicMax(&fb[1], w + 1); }
}
// the null words of many columns in one launch (fb: [0] nulls, [1] last non-zero word + 1): blockIdx.y = column, a
// grid-stride loop over its words
struct NullJob { const uint8_t* nulls; uint64_t* words; int* fb; int n; int pad_; };
__global__ void enc_null_words_many_kernel(const NullJob* jobs) {
  const NullJob j = jobs[blockIdx.y];
  for (int w = blockIdx.x * blockDim.x + threadIdx.x; (int64_t)w * 64 < j.n; w += gridDim.x * blockDim.x) null_word(j.nulls, j.n, j.words, j.fb, w);
}

template <class T> __device__ __forceinline__ T ld_raw(const uint8_t* p, int64_t i) { return reinterpret_cast<const T*>(p)[i]; }

// one CTA per column: tiles of 1024 rows, block-wide exclusive scan of the non-null flags, values scattered to their
// compacted position; min / max on the way (the stats row's lower / upper bounds)
template <int KIND>
__device__ void enc_compact(const EncCol& c) {
  __shared__ int warp_sum[32];
  __shared__ int tile_base;
  __shared__ unsigned long long red_lo[32], red_hi[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) tile_base = 0;
  __syncthreads();
  double dlo = 0, dhi = 0;
  long long ilo = LLONG_MAX, ihi = LLONG_MIN;
  bool have = false;
  for (int t0 = 0; t0 < c.n; t0 += 1024) {
    const int i = t0 + tid;
    const bool valid = i < c.n && !(c.nulls && c.nulls[i]);
    const unsigned m = __ballot_sync(0xffffffffu, valid);
    if (lane == 0) warp_sum[warp] = __popc(m);
    __syncthreads();
    int before = __popc(m & ((1u << lane) - 1u));
    for (int w = 0; w < warp; w++) before += warp_sum[w];
    const int64_t k = (int64_t)tile_base + before;
    if (valid) {
      if (KIND == EK_I8) { const int8_t v = ld_raw<int8_t>(c.values, i); reinterpret_cast<int8_t*>(c.out)[k] = v; ilo = min(ilo, (long long)v); ihi = max(ihi, (long long)v); }
      else if (KIND == EK_I16) { const int16_t v = ld_raw<int16_t>(c.values, i); reinterpret_cast<int16_t*>(c.out)[k] = v; ilo = min(ilo, (long long)v); ihi = max(ihi, (long long)v); }
      else if (KIND == EK_I32) { const int32_t v = ld_raw<int32_t>(c.values, i); reinterpret_cast<int32_t*>(c.out)[k] = v; ilo = min(ilo, (long long)v); ihi = max(ihi, (long long)v); }
      else if (KIND == EK_I64) { const int64_t v = ld_raw<int64_t>(c.values, i); reinterpret_cast<int64_t*>(c.out)[k] = v; ilo = min(ilo, (long long)v); ihi = max(ihi, (long long)v); }
      else if (KIND == EK_F32) { const float v = ld_raw<float>(c.values, i); reinterpret_cast<float*>(c.out)[k] = v; if (!have) { dlo = dhi = v; } else { dlo = fmin(dlo, (double)v); dhi = fmax(dhi, (double)v); } }
      else if (KIND == EK_F64) { const double v = ld_raw<double>(c.values, i); reinterpret_cast<double*>(c.out)[k] = v; if (!have) { dlo = dhi = v; } else { dlo = fmin(dlo, v); dhi = fmax(dhi, v); } }
      else if (KIND == EK_BOOL) {   // bit k of the LE 64-bit words = k-th non-null value (enc/BooleanBitSetEncoding.scala:62-152)
        const long long v = c.values[i] != 0;
        if (v) atomicOr(reinterpret_cast<unsigned int*>(c.out) + (k >> 5), 1u << (k & 31));
        ilo = min(ilo, v); ihi = max(ihi, v);
      } else if (KIND == EK_STRCODE16) reinterpret_cast<int16_t*>(c.out)[k] = (int16_t)c.slot_code[ld_raw<int32_t>(c.values, i)];
      else reinterpret_cast<int32_t*>(c.out)[k] = c.slot_code[ld_raw<int32_t>(c.values, i)];
      have = true;
    }
    __syncthreads();
    if (tid == 0) { int tot = 0; for (int w = 0; w < 32; w++) tot += warp_sum[w]; tile_base += tot; }
    __syncthreads();
  }
  // bounds: block reduction (first non-null value seeds the floating-point pair)
  const bool fp = KIND == EK_F32 || KIND == EK_F64;
  unsigned long long lo_bits, hi_bits;
  if (fp) {
    double a = have ? dlo : __longlong_as_double(0x7ff0000000000000ll), b = have ? dhi : __longlong_as_double(0xfff0000000000000ll);
    for (int d = 16; d > 0; d >>= 1) { a = fmin(a, __shfl_xor_sync(0xffffffffu, a, d)); b = fmax(b, __shfl_xor_sync(0xffffffffu, b, d)); }
    lo_bits = (unsigned long long)__double_as_longlong(a); hi_bits = (unsigned long long)__double_as_longlong(b);
  } else {
    long long a = ilo, b = ihi;
    for (int d = 16; d > 0; d >>= 1) { a = min(a, __shfl_xor_sync(0xffffffffu, a, d)); b = max(b, __shfl_xor_sync(0xffffffffu, b, d)); }
    lo_bits = (unsigned long long)a; hi_bits = (unsigned long long)b;
  }
  if (lane == 0) { red_lo[warp] = lo_bits; red_hi[warp] = hi_bits; }
  __syncthreads();
  if (tid == 0) {
    if (fp) {
      double a = __longlong_as_double((long long)red_lo[0]), b = __longlong_as_double((long long)red_hi[0]);
      for (int w = 1; w < 32; w++) { a = fmin(a, __longlong_as_double((long long)red_lo[w])); b = fmax(b, __longlong_as_double((long long)red_hi[w])); }
      c.stat[0] = (uint64_t)__double_as_longlong(a); c.stat[1] = (uint64_t)__double_as_longlong(b);
    } else {
      long long a = (long long)red_lo[0], b = (long long)red_hi[0];
      for (int w = 1; w < 32; w++) { a = min(a, (long long)red_lo[w]); b = max(b, (long long)red_hi[w]); }
      c.stat[0] = (uint64_t)a; c.stat[1] = (uint64_t)b;
    }
    c.stat[2] = (uint64_t)tile_base;
  }
}

__global__ void __launch_bounds__(1024) enc_compact_kernel(const EncCol* cols) {
  const EncCol& c = cols[blockIdx.x];
  switch (c.kind) {
    case EK_I8: enc_compact<EK_I8>(c); break;
    case EK_I16: enc_compact<EK_I16>(c); break;
    case EK_I32: enc_compact<EK_I32>(c); break;
    case EK_I64: enc_compact<EK_I64>(c); break;
    case EK_F32: enc_compact<EK_F32>(c); break;
    case EK_F64: enc_compact<EK_F64>(c); break;
    case EK_BOOL: enc_compact<EK_BOOL>(c); break;
    case EK_STRCODE16: enc_compact<EK_STRCODE16>(c); break;
    default: enc_compact<EK_STRCODE32>(c); break;
  }
}

// ---- distinct strings and their first occurrence (DictionaryEncoder hands out indexes in insertion order) ------------
// open addressing over row ordinals: slot = smallest row seen so far among the rows with these bytes (-1: empty)
__device__ __forceinline__ bool str_rows_equal(const int32_t* offs, const uint8_t* bytes, int a, int b) {
  const int la = offs[a + 1] - offs[a];
  if (la != offs[b + 1] - offs[b]) return false;
  const uint8_t *pa = bytes + offs[a], *pb = bytes + offs[b];
  for (int i = 0; i < la; i++) if (pa[i] != pb[i]) return false;
  return true;
}
__global__ void dict_insert_kernel(const int32_t* offs, const uint8_t* bytes, const uint8_t* nulls, int n, int* slots, uint32_t mask,
                                   int32_t* slot_of_row) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (nulls && nulls[i]) { slot_of_row[i] = -1; continue; }
    uint64_t h = 1469598103934665603ull;
    for (int k = offs[i]; k < offs[i + 1]; k++) { h ^= bytes[k]; h *= 1099511628211ull; }
    uint32_t pos = (uint32_t)(h ^ (h >> 32)) & mask;
    for (;;) {
      int r = atomicCAS(&slots[pos], -1, i);
      if (r == -1) break;                                             // claimed an empty slot
      if (str_rows_equal(offs, bytes, r, i)) { atomicMin(&slots[pos], i); break; }   // same string: keep the earliest row
      pos = (pos + 1) & mask;
    }
    slot_of_row[i] = (int32_t)pos;
  }
}
__global__ void dict_collect_kernel(const int* slots, uint32_t cap, int2* out, int* count) {
  for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < cap; s += gridDim.x * blockDim.x)
    if (slots[s] >= 0) { const int k = atomicAdd(count, 1); out[k] = make_int2((int)s, slots[s]); }
}
__global__ void dict_codes_kernel(const int2* pairs, int n, int32_t* slot_code) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) slot_code[pairs[k].x] = pairs[k].y;
}

int width_of(int t) {
  switch (t) {
    case SD_BOOLEAN: case SD_BYTE: return 1;
    case SD_SHORT: return 2;
    case SD_INT: case SD_DATE: case SD_FLOAT: return 4;
    case SD_LONG: case SD_TIMESTAMP: case SD_DOUBLE: case SD_DECIMAL: return 8;
  }
  return 0;
}
int kind_of(int t) {
  switch (t) {
    case SD_BOOLEAN: return EK_BOOL; case SD_BYTE: return EK_I8; case SD_SHORT: return EK_I16;
    case SD_INT: case SD_DATE: return EK_I32; case SD_FLOAT: return EK_F32; case SD_DOUBLE: return EK_F64;
    default: return EK_I64;
  }
}
void put32(std::vector<uint8_t>& b, int32_t v) { b.insert(b.end(), reinterpret_cast<uint8_t*>(&v), reinterpret_cast<uint8_t*>(&v) + 4); }

}  // namespace

namespace {
// entry f.. of a stats row: (lower, upper, nullCount) of one column, written over whatever the slots held; STRING bounds go
// to the end of the variable-length region
void put_entry(std::vector<uint8_t>& row, int64_t bits, int f, const ColStat& s) {
  auto setnull = [&](int i, bool v) { if (v) row[i >> 3] |= (uint8_t)(1u << (i & 7)); else row[i >> 3] &= (uint8_t)~(1u << (i & 7)); };
  auto slot = [&](int i) { return row.data() + bits + 8ll * i; };
  for (int k = 0; k < 3; k++) { memset(slot(f + k), 0, 8); setnull(f + k, !s.present); }
  if (!s.present) return;
  memcpy(slot(f + 2), &s.nulls, 4);
  if (!s.has) { setnull(f, true); setnull(f + 1, true); return; }
  for (int w = 0; w < 2; w++) {
    if (s.type == SD_STRING) {
      const std::string& v = w ? s.shi : s.slo;
      const int64_t ol = ((int64_t)row.size() << 32) | (int64_t)v.size();
      memcpy(slot(f + w), &ol, 8);
      row.insert(row.end(), v.begin(), v.end());
      while (row.size() % 8) row.push_back(0);
    } else {
      const uint64_t raw = w ? s.hi : s.lo;
      switch (s.type) {
        case SD_BOOLEAN: *slot(f + w) = raw != 0; break;
        case SD_BYTE: memcpy(slot(f + w), &raw, 1); break;
        case SD_SHORT: memcpy(slot(f + w), &raw, 2); break;
        case SD_INT: case SD_DATE: memcpy(slot(f + w), &raw, 4); break;
        case SD_FLOAT: { double d; memcpy(&d, &raw, 8); float fl = (float)d; memcpy(slot(f + w), &fl, 4); break; }
        default: memcpy(slot(f + w), &raw, 8); break;
      }
    }
  }
}
int64_t stats_bits(int ncols) { return (int64_t)((1 + 3 * ncols + 63) / 64) * 8; }
}  // namespace

std::vector<uint8_t> stats_row_bytes(int32_t count, const std::vector<ColStat>& st) {
  const int nf = 1 + 3 * (int)st.size();
  const int64_t bits = stats_bits((int)st.size()), fixed = bits + 8ll * nf;
  std::vector<uint8_t> row((size_t)fixed, 0);
  memcpy(row.data() + bits, &count, 4);
  for (size_t c = 0; c < st.size(); c++) put_entry(row, bits, 1 + 3 * (int)c, st[c]);
  return row;
}

void stats_row_replace(std::vector<uint8_t>& row, int ncols, int32_t count, const std::vector<std::pair<int, const ColStat*>>& entries) {
  const int64_t bits = stats_bits(ncols);
  if ((int64_t)row.size() < bits + 8ll * (1 + 3 * ncols)) return;   // not a stats row of ncols columns: left alone
  memset(row.data() + bits, 0, 8);
  memcpy(row.data() + bits, &count, 4);
  for (auto& e : entries)
    if (e.first < ncols) put_entry(row, bits, 1 + 3 * e.first, *e.second);
}

void enc_first_seen_dict(EncJob& j, std::vector<int2>& slot_first, const std::function<std::string(int slot, int first)>& value_of) {
  std::sort(slot_first.begin(), slot_first.end(), [](const int2& a, const int2& b) { return a.y < b.y || (a.y == b.y && a.x < b.x); });
  j.dict.clear();
  j.slot_codes.clear();
  for (size_t d = 0; d < slot_first.size(); d++) {
    j.dict.push_back(value_of(slot_first[d].x, slot_first[d].y));
    j.slot_codes.push_back(make_int2(slot_first[d].x, (int)d));
  }
}

bool enc_queue_words(cudaStream_t st, const std::vector<EncJob*>& jobs, int* rc) {
  bool any = false;
  *rc = 0;
  for (EncJob* j : jobs) {
    if (j->fb[1] <= 0) continue;
    j->words.resize((size_t)j->fb[1]);
    const cudaError_t e = cudaMemcpyAsync(j->words.data(), j->d_words, (size_t)j->fb[1] * 8, cudaMemcpyDeviceToHost, st);
    if (e != cudaSuccess) { *rc = set_error(SD_ERR_CUDA, "null words read-back failed: %s", cudaGetErrorString(e)); return any; }
    any = true;
  }
  return any;
}

int enc_null_words_many(cudaStream_t st, const std::vector<EncJob*>& jobs, DevAllocFn alloc, void* ctx, PinnedArena& pin) {
  std::vector<NullJob> nj;
  int max_words = 0;
  for (EncJob* j : jobs) {
    if (!j->d_nulls || j->n <= 0) continue;
    nj.push_back(NullJob{j->d_nulls, j->d_words, j->d_fb, j->n, 0});
    max_words = std::max(max_words, (j->n + 63) / 64);
  }
  for (size_t at = 0; at < nj.size(); at += 65535) {   // gridDim.y limit
    const size_t cnt = std::min<size_t>(65535, nj.size() - at);
    uint8_t* h = pin.alloc(cnt * sizeof(NullJob));
    uint8_t* d = alloc(ctx, cnt * sizeof(NullJob));
    if (!h || !d) return SD_ERR_CUDA;
    memcpy(h, nj.data() + at, cnt * sizeof(NullJob));
    SD_CUDA(cudaMemcpyAsync(d, h, cnt * sizeof(NullJob), cudaMemcpyHostToDevice, st));
    enc_null_words_many_kernel<<<dim3((unsigned)std::min(64, (max_words + 255) / 256), (unsigned)cnt), 256, 0, st>>>(reinterpret_cast<const NullJob*>(d));
    SD_CUDA(cudaGetLastError());
  }
  return 0;
}

int enc_layout(sd_store* s, cudaStream_t st, PinnedArena& pin, EncJob& j, StoredCol& sc, ColStat& cs) {
  const int nn = j.n - j.fb[0];
  std::vector<uint8_t> pre;
  int type_id = ENC_UNCOMPRESSED;
  cs = ColStat();
  if (j.type == SD_STRING) {
    const int nd = (int)j.dict.size();
    const bool big = nd > 32767;   // index Short.MaxValue switches to int32 indexes (enc/DictionaryEncoding.scala:313-318)
    type_id = big ? ENC_BIG_DICTIONARY : ENC_DICTIONARY;
    put32(pre, type_id); put32(pre, (int32_t)j.words.size() * 8);
    pre.insert(pre.end(), reinterpret_cast<uint8_t*>(j.words.data()), reinterpret_cast<uint8_t*>(j.words.data()) + j.words.size() * 8);
    put32(pre, nd);
    for (const std::string& sv : j.dict) {
      put32(pre, (int32_t)sv.size());
      pre.insert(pre.end(), sv.begin(), sv.end());
      if (!cs.has || sv < cs.slo) cs.slo = sv;      // std::string compares as unsigned bytes, shorter first on a common prefix
      if (!cs.has || sv > cs.shi) cs.shi = sv;
      cs.has = true;
    }
    j.body_len = (int64_t)nn * (big ? 4 : 2);
  } else {
    type_id = j.type == SD_BOOLEAN ? ENC_BOOLEAN_BITSET : ENC_UNCOMPRESSED;
    put32(pre, type_id); put32(pre, (int32_t)j.words.size() * 8);
    pre.insert(pre.end(), reinterpret_cast<uint8_t*>(j.words.data()), reinterpret_cast<uint8_t*>(j.words.data()) + j.words.size() * 8);
    j.body_len = j.type == SD_BOOLEAN ? ((int64_t)(nn + 63) / 64) * 8 : (int64_t)nn * width_of(j.type);
    cs.has = nn > 0;
  }
  int rc = store_register_encoded(s, pre.data(), (int64_t)pre.size(), (int64_t)pre.size() + j.body_len, j.type, j.nullable ? 1 : 0, j.n, sc);
  if (rc) return rc;
  uint8_t* h_pre = pin.alloc(pre.size());   // page-locked staging (stays valid until the stream has drained)
  if (!h_pre) return SD_ERR_CUDA;
  memcpy(h_pre, pre.data(), pre.size());
  SD_CUDA(cudaMemcpyAsync(sc.dev_base, h_pre, pre.size(), cudaMemcpyHostToDevice, st));
  j.d_body = sc.dev_base + pre.size();
  if (j.type == SD_STRING && !j.slot_codes.empty()) {
    uint8_t* h_pairs = pin.alloc(j.slot_codes.size() * 8);
    if (!h_pairs) return SD_ERR_CUDA;
    memcpy(h_pairs, j.slot_codes.data(), j.slot_codes.size() * 8);
    SD_CUDA(cudaMemcpyAsync(j.d_slot_pairs, h_pairs, j.slot_codes.size() * 8, cudaMemcpyHostToDevice, st));
    dict_codes_kernel<<<((int)j.slot_codes.size() + 255) / 256, 256, 0, st>>>(j.d_slot_pairs, (int)j.slot_codes.size(), j.d_slot_code);
    SD_CUDA(cudaGetLastError());
  }
  if (j.type == SD_BOOLEAN && j.body_len) SD_CUDA(cudaMemsetAsync(j.d_body, 0, (size_t)j.body_len, st));
  cs.present = true; cs.type = j.type; cs.nulls = j.fb[0];
  return 0;
}

int enc_write(cudaStream_t st, DevAllocFn alloc, void* ctx, PinnedArena& pin, const std::vector<EncJob*>& jobs, const std::vector<ColStat*>& stats,
              cudaEvent_t ev_begin, cudaEvent_t ev_end) {
  if (jobs.empty()) return 0;
  std::vector<EncCol> enc(jobs.size());
  for (size_t k = 0; k < jobs.size(); k++) {
    const EncJob& j = *jobs[k];
    EncCol& e = enc[k];
    memset(&e, 0, sizeof(e));
    e.nulls = j.d_nulls; e.out = j.d_body; e.stat = j.d_stat; e.n = j.n;
    if (j.type == SD_STRING) {
      e.values = j.d_values;
      e.kind = j.dict.size() > 32767 ? EK_STRCODE32 : EK_STRCODE16;
      e.slot_code = j.d_slot_code;
    } else {
      e.values = j.d_values;
      e.kind = kind_of(j.type);
    }
  }
  uint8_t* d_enc = alloc(ctx, enc.size() * sizeof(EncCol) + 64);
  uint8_t* h_enc = pin.alloc(enc.size() * sizeof(EncCol));
  if (!d_enc || !h_enc) return SD_ERR_CUDA;
  memcpy(h_enc, enc.data(), enc.size() * sizeof(EncCol));
  SD_CUDA(cudaMemcpyAsync(d_enc, h_enc, enc.size() * sizeof(EncCol), cudaMemcpyHostToDevice, st));
  if (ev_begin) SD_CUDA(cudaEventRecord(ev_begin, st));
  enc_compact_kernel<<<(int)enc.size(), 1024, 0, st>>>(reinterpret_cast<const EncCol*>(d_enc));
  SD_CUDA(cudaGetLastError());
  if (ev_end) SD_CUDA(cudaEventRecord(ev_end, st));
  std::vector<uint64_t> hst(jobs.size() * 3);
  for (size_t k = 0; k < jobs.size(); k++) SD_CUDA(cudaMemcpyAsync(&hst[3 * k], jobs[k]->d_stat, 24, cudaMemcpyDeviceToHost, st));
  SD_CUDA(cudaStreamSynchronize(st));
  for (size_t k = 0; k < jobs.size(); k++) {
    ColStat& cs = *stats[k];
    if (jobs[k]->type != SD_STRING && cs.has) { cs.lo = hst[3 * k]; cs.hi = hst[3 * k + 1]; }
    if ((int64_t)hst[3 * k + 2] != (int64_t)(jobs[k]->n - jobs[k]->fb[0])) return set_error(SD_ERR_CUDA, "encoder: non-null count mismatch in column %d", jobs[k]->table_col);
  }
  return 0;
}

}  // namespace sd

extern "C" int sd_store_encode_batch(sd_store* s, int32_t num_rows, const sd_raw_column* cols, int32_t ncols, int32_t bucket_id, int64_t batch_id) {
  using namespace sd;
  if (!s || !cols || num_rows < 0) return set_error(SD_ERR_INVALID, "sd_store_encode_batch: bad arguments");
  if (ncols != (int)s->schema.size()) return set_error(SD_ERR_INVALID, "sd_store_encode_batch: %d columns, table schema has %zu", ncols, s->schema.size());
  // Scans of the store go on while a batch is being encoded: the store's lock is held only to lay the buffers out in the
  // arena (phase 2) and to publish the finished batch; everything that touches the rows runs on the encoder's own stream.
  std::lock_guard<std::mutex> enc_lock(s->enc_mu);
  SD_CUDA(cudaSetDevice(s->device));
  if (!s->enc_stream) {
    SD_CUDA(cudaStreamCreateWithFlags(&s->enc_stream, cudaStreamNonBlocking));
    SD_CUDA(cudaEventCreateWithFlags(&s->enc_event, cudaEventDisableTiming));
  }
  cudaStream_t st = s->enc_stream;
  int64_t h2d = 0;
  const int n = num_rows;
  Arena tmp;
  tmp.device = s->device;
  tmp.slab_bytes = size_t(64) << 20;
  const DevAllocFn tmp_alloc = [](void* a, size_t bytes) { return reinterpret_cast<Arena*>(a)->alloc(bytes, 16); };
  auto to_dev = [&](const void* src, size_t bytes, size_t align, uint8_t** out) -> int {
    uint8_t* d = tmp.alloc(bytes + 64, align);
    if (!d) return SD_ERR_CUDA;
    if (bytes) SD_CUDA(cudaMemcpyAsync(d, src, bytes, cudaMemcpyHostToDevice, st));
    h2d += (int64_t)bytes;
    *out = d;
    return 0;
  };
  struct Work {
    EncJob job;
    uint8_t* d_bytes = nullptr;   // STRING: the values' bytes
    int* d_slots = nullptr; int* d_count = nullptr; int2* d_pairs = nullptr; uint32_t cap = 0;
  };
  std::vector<Work> work;
  for (int c = 0; c < ncols; c++)   // before anything is copied: the store stays unchanged
    if (cols[c].values && wide_decimal(s->schema[c].type, s->schema[c].precision))
      return set_error(SD_ERR_UNSUPPORTED, "column %d: DECIMAL(%d,%d) is wider than 18 digits: the device encoder writes int64 unscaled values only", c,
                       s->schema[c].precision, s->schema[c].scale);
  // ---- phase 1: raw values to the device; null words; distinct strings -------------------------------------------------
  for (int c = 0; c < ncols; c++) {
    if (!cols[c].values) continue;
    Work w;
    EncJob& j = w.job;
    j.table_col = c; j.type = s->schema[c].type; j.nullable = s->schema[c].nullable != 0; j.n = n;
    if (cols[c].nulls && !j.nullable) return set_error(SD_ERR_INVALID, "column %d is NOT NULL but a null mask was given", c);
    int rc = 0;
    uint8_t* d_values = nullptr;
    if (j.type == SD_STRING) {
      const int32_t* offs = reinterpret_cast<const int32_t*>(cols[c].values);
      if (!cols[c].str_bytes && n > 0 && offs[n] > 0) return set_error(SD_ERR_INVALID, "column %d: STRING column without bytes", c);
      rc = to_dev(offs, (size_t)(n + 1) * 4, 16, &d_values);
      if (!rc) rc = to_dev(cols[c].str_bytes, n > 0 ? (size_t)offs[n] : 0, 16, &w.d_bytes);
    } else {
      const int wd = width_of(j.type);
      if (!wd) return set_error(SD_ERR_UNSUPPORTED, "column %d: type %d cannot be encoded", c, j.type);
      rc = to_dev(cols[c].values, (size_t)n * wd, 16, &d_values);
    }
    if (rc) return rc;
    j.d_values = d_values;
    if (cols[c].nulls) {
      uint8_t* d_nulls = nullptr;
      rc = to_dev(cols[c].nulls, (size_t)n, 16, &d_nulls);
      if (rc) return rc;
      j.d_nulls = d_nulls;
    }
    j.d_stat = reinterpret_cast<uint64_t*>(tmp.alloc(64, 16));
    j.d_fb = reinterpret_cast<int*>(tmp.alloc(64, 16));
    if (!j.d_stat || !j.d_fb) return SD_ERR_CUDA;
    SD_CUDA(cudaMemsetAsync(j.d_fb, 0, 64, st));
    if (j.d_nulls && n > 0) {
      const int nw = (n + 63) / 64;
      j.d_words = reinterpret_cast<uint64_t*>(tmp.alloc((size_t)nw * 8 + 64, 16));
      if (!j.d_words) return SD_ERR_CUDA;
    }
    if (j.type == SD_STRING && n > 0) {
      w.cap = 1024;
      while (w.cap < 2u * (uint32_t)n) w.cap <<= 1;
      w.d_slots = reinterpret_cast<int*>(tmp.alloc((size_t)w.cap * 4, 16));
      j.d_slot_code = reinterpret_cast<int32_t*>(tmp.alloc((size_t)w.cap * 4, 16));
      int32_t* d_slot_of_row = reinterpret_cast<int32_t*>(tmp.alloc((size_t)n * 4 + 64, 16));
      w.d_pairs = reinterpret_cast<int2*>(tmp.alloc((size_t)n * 8 + 64, 16));
      w.d_count = reinterpret_cast<int*>(tmp.alloc(64, 16));
      if (!w.d_slots || !j.d_slot_code || !d_slot_of_row || !w.d_pairs || !w.d_count) return SD_ERR_CUDA;
      SD_CUDA(cudaMemsetAsync(w.d_slots, 0xff, (size_t)w.cap * 4, st));
      SD_CUDA(cudaMemsetAsync(w.d_count, 0, 4, st));
      dict_insert_kernel<<<592, 256, 0, st>>>(reinterpret_cast<const int32_t*>(d_values), w.d_bytes, j.d_nulls, n, w.d_slots, w.cap - 1, d_slot_of_row);
      SD_CUDA(cudaGetLastError());
      dict_collect_kernel<<<592, 256, 0, st>>>(w.d_slots, w.cap, w.d_pairs, w.d_count);
      SD_CUDA(cudaGetLastError());
      j.d_values = reinterpret_cast<const uint8_t*>(d_slot_of_row);   // the encoder reads the slot of every row
      j.d_slot_pairs = w.d_pairs;
    }
    work.push_back(std::move(w));
  }
  std::vector<EncJob*> jobs;
  for (Work& w : work) jobs.push_back(&w.job);
  {
    int rc = enc_null_words_many(st, jobs, tmp_alloc, &tmp, s->enc_host);
    if (rc) return rc;
  }
  // ---- feedback: null counts / trimmed word counts / null words, distinct strings ----------------------------------------
  std::vector<std::vector<int2>> pairs(work.size());
  std::vector<int> ndistinct(work.size(), 0);
  for (size_t k = 0; k < work.size(); k++) {
    Work& w = work[k];
    SD_CUDA(cudaMemcpyAsync(w.job.fb, w.job.d_fb, 8, cudaMemcpyDeviceToHost, st));
    if (w.d_count) SD_CUDA(cudaMemcpyAsync(&ndistinct[k], w.d_count, 4, cudaMemcpyDeviceToHost, st));
  }
  SD_CUDA(cudaStreamSynchronize(st));
  {
    int rc = 0;
    enc_queue_words(st, jobs, &rc);
    if (rc) return rc;
  }
  for (size_t k = 0; k < work.size(); k++) {
    if (ndistinct[k] > 0) { pairs[k].resize((size_t)ndistinct[k]); SD_CUDA(cudaMemcpyAsync(pairs[k].data(), work[k].d_pairs, (size_t)ndistinct[k] * 8, cudaMemcpyDeviceToHost, st)); }
  }
  SD_CUDA(cudaStreamSynchronize(st));
  // dictionary in first-seen order: the distinct strings by the earliest row that holds them
  for (size_t k = 0; k < work.size(); k++) {
    EncJob& j = work[k].job;
    if (j.type != SD_STRING) continue;
    const int32_t* offs = reinterpret_cast<const int32_t*>(cols[j.table_col].values);
    const uint8_t* bytes = cols[j.table_col].str_bytes;
    enc_first_seen_dict(j, pairs[k], [&](int, int row) {
      return std::string(reinterpret_cast<const char*>(bytes + offs[row]), (size_t)(offs[row + 1] - offs[row]));
    });
  }
  // ---- layout on the host; registration in the store; phase 2 ----------------------------------------------------------
  std::unique_ptr<StoredBatch> sb(new StoredBatch());
  sb->num_rows = n; sb->bucket_id = bucket_id; sb->batch_id = batch_id;
  sb->cols.resize(s->schema.size());
  std::vector<ColStat> stats(s->schema.size());
  std::vector<ColStat*> job_stats;
  std::unique_lock<std::mutex> store_lock(s->mu);   // phase 2: arena placement + the small side uploads of upload_column
  {
    ExtentRecorder rec(s->arena, &sb->extents);
    for (Work& w : work) {
      int rc = enc_layout(s, st, s->enc_host, w.job, sb->cols[w.job.table_col], stats[w.job.table_col]);
      if (rc) return rc;
      job_stats.push_back(&stats[w.job.table_col]);
    }
  }
  // the side uploads (null words, prefixes of "nulls before") went over the store's copy stream: order the encoder after them
  SD_CUDA(cudaEventRecord(s->enc_event, s->copy_stream));
  SD_CUDA(cudaStreamWaitEvent(st, s->enc_event, 0));
  store_lock.unlock();
  {
    int rc = enc_write(st, tmp_alloc, &tmp, s->enc_host, jobs, job_stats);
    if (rc) return rc;
  }
  sb->stats = stats_row_bytes(n, stats);
  sb->stats_ncols = (int32_t)s->schema.size();
  SD_CUDA(cudaStreamSynchronize(st));   // bodies written, side uploads done (ordered above): the batch may become visible
  {
    int rc = build_images(s, st, {sb.get()}, false);
    if (rc) return rc;
  }
  {
    std::lock_guard<std::mutex> lock(s->mu);
    s->batches.push_back(std::move(sb));
    s->version++;
    s->h2d_bytes += h2d;
  }
  s->enc_host.reset();
  return 0;   // `tmp` (the raw values' staging) is released here; everything queued on the stream has completed
}

// the stats row the encoder produced for a resident batch (tests compare it with the fixture writer's)
extern "C" int sdx_store_get_stats(sd_store* s, int64_t batch_index, void* out, int64_t cap, int64_t* out_len) {
  using namespace sd;
  if (!s || !out_len) return set_error(SD_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lock(s->mu);
  if (batch_index < 0 || batch_index >= (int64_t)s->batches.size()) return set_error(SD_ERR_INVALID, "batch index out of range");
  const std::vector<uint8_t>& st = s->batches[batch_index]->stats;
  *out_len = (int64_t)st.size();
  if ((int64_t)st.size() > cap) return set_error(SD_ERR_OVERFLOW, "buffer too small");
  if (!st.empty()) memcpy(out, st.data(), st.size());
  return 0;
}
