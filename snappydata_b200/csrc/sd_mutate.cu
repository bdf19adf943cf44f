// sd_mutate.cu -- UPDATE / DELETE over a resident store, on the device: the write side of the reference's ColumnUpdateExec /
// ColumnDeleteExec (core/.../columnar/ColumnUpdateExec.scala, ColumnDeleteExec.scala) together with the store-side merge that
// ColumnDelta.apply performs when the new delta is put (encoders/.../impl/ColumnDelta.scala:64-222).
//
//   1. scan    the plan (MODE_MUTATE) emits one record per matching live row: (batch, row) key, SET null bits, SET values
//              (sd_engine.cu mutation_scan: staged ring, overlay path, stats skipping, grow-and-replay);
//   2. sort    the records by (batch ordinal, row) with a CUB radix sort of the 64-bit key (a row is scanned once, so the
//              positions of one batch are unique);
//   3. count   one CTA per (batch, SET target) pair -- per batch for a DELETE -- sizes the merge of the new positions with the
//              existing depth-0 delta (delete mask): union size, NULLs, bounds of the new values.  One read-back;
//   4. layout  the host places every output in the store's arena, all at once for the statement;
//   5. write   the same CTAs write the merged delta in the reference's layout (ColumnDeltaEncoder.merge,
//              enc/ColumnDeltaEncoder.scala:348-556: union of positions, the NEW value wins on an equal position, re-encoded
//              Uncompressed) or the merged delete mask (ColumnDeleteEncoder.merge: ascending union);
//   6. install new StoredBatch versions (new uid) under the store's lock, all of the statement's at once.
//
// The merge is rank based: the output slot of an entry is its index in its own list plus the number of entries of the other
// list below it, less the duplicates, so every thread of a CTA places its entries independently (binary searches + one
// block-wide scan per tile of entries).
#include <cub/cub.cuh>

#include <algorithm>
#include <chrono>
#include <cstring>
#include <unordered_map>

#include "sd_host.h"

namespace sd {
namespace {

constexpr int MT = 256;   // threads of the merge kernels

// one (batch, SET target) pair of an UPDATE, or one batch of a DELETE (slot = -1)
struct MergePair {
  int32_t batch;           // ordinal in the statement's batch list
  int32_t slot;            // SET value index in the record; -1: DELETE
  int32_t type;            // sd_type of the target column
  int32_t width;           // bytes per stored value
  const int32_t* ex_pos;   // existing depth-0 delta / delete mask: ascending positions
  const uint64_t* ex_nulls;
  const uint8_t* ex_data;  // values (Uncompressed) or dictionary indexes
  const uint8_t* ex_dict;  // INT / LONG dictionary of a Dictionary-encoded delta
  int32_t ex_n;
  int32_t ex_nwords;
  int32_t ex_enc;
  int32_t pad_;
  int64_t scratch_off;     // this pair's [n_new + 1] duplicate prefix: scratch[scratch_off + first record of the batch ...]
  int32_t* out_pos;        // write pass: the merged positions ...
  uint64_t* out_nulls;     // ... null words (trimmed) ...
  uint8_t* out_vals;       // ... and the non-null values
  uint64_t* tmp_val;       // [union] merged raw values before compaction
  uint8_t* tmp_null;       // [union] merged null flags
};

struct PairCounts {
  int64_t n_new, n_union, union_nulls, new_nulls, max_null_idx;
  uint64_t new_min, new_max;   // order-preserving keys of the new non-null values (see value_key)
  int64_t pad_;
};

__device__ __forceinline__ int lower_bound_i32(const int32_t* a, int n, int32_t v) {
  int lo = 0, hi = n;
  while (lo < hi) { const int m = (lo + hi) >> 1; if (a[m] < v) lo = m + 1; else hi = m; }
  return lo;
}
__device__ __forceinline__ int lower_bound_key(const uint64_t* a, int n, uint32_t v) {   // on the row half of sorted keys
  int lo = 0, hi = n;
  while (lo < hi) { const int m = (lo + hi) >> 1; if ((uint32_t)a[m] < v) lo = m + 1; else hi = m; }
  return lo;
}

__device__ __forceinline__ bool is_fp(int t) { return t == SD_FLOAT || t == SD_DOUBLE; }

// an order-preserving unsigned key of a value: integral values as offset binary, floating point in the total order of
// java.lang.Double.compare (what the stats row's interpreted ordering uses; one NaN, the greatest)
__device__ __forceinline__ uint64_t value_key(int type, uint64_t raw) {
  if (!is_fp(type)) return raw ^ 0x8000000000000000ull;
  double d = __longlong_as_double((long long)raw);
  uint64_t b = d != d ? 0x7ff8000000000000ull : raw;
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

// the new entry's value as raw bits of the target's stored width (records hold integral values sign-extended to 64 bits and
// floating point values as doubles)
__device__ __forceinline__ uint64_t stored_bits(int type, uint64_t rec_val) {
  if (type == SD_FLOAT) { const float f = (float)__longlong_as_double((long long)rec_val); return (uint64_t)__float_as_uint(f); }
  return rec_val;
}
// an existing delta's value j (value index vi) -> raw stored bits, and as a record-style value for the bounds
__device__ __forceinline__ uint64_t existing_bits(const MergePair& p, int vi) {
  if (p.ex_enc == ENC_UNCOMPRESSED) {
    uint64_t v = 0;
    const uint8_t* q = p.ex_data + (size_t)vi * p.width;
    for (int k = 0; k < p.width; k++) v |= (uint64_t)q[k] << (8 * k);
    return v;
  }
  const int idx = p.ex_enc == ENC_DICTIONARY ? (int)reinterpret_cast<const int16_t*>(p.ex_data)[vi] : reinterpret_cast<const int32_t*>(p.ex_data)[vi];
  if (p.width == 4) return (uint64_t)reinterpret_cast<const uint32_t*>(p.ex_dict)[idx];
  return reinterpret_cast<const uint64_t*>(p.ex_dict)[idx];
}

template <bool WRITE>
__global__ void __launch_bounds__(MT) merge_kernel(const MergePair* __restrict__ pairs, const uint64_t* __restrict__ keys,
                                                   const uint32_t* __restrict__ order, const uint64_t* __restrict__ recs, int rec_words,
                                                   const int32_t* __restrict__ seg, int32_t* __restrict__ scratch, PairCounts* counts) {
  typedef cub::BlockScan<int, MT> Scan;
  typedef cub::BlockReduce<long long, MT> RedI;
  typedef cub::BlockReduce<unsigned long long, MT> RedU;
  __shared__ union { typename Scan::TempStorage scan; typename RedI::TempStorage ri; typename RedU::TempStorage ru; } tmp;
  __shared__ int carry;
  const MergePair p = pairs[blockIdx.x];
  const int tid = threadIdx.x;
  const int lo = seg[2 * p.batch], n_new = seg[2 * p.batch + 1] - lo;
  if (n_new <= 0) {
    if (!WRITE && tid == 0) { PairCounts c = {}; c.max_null_idx = -1; c.new_min = ~0ull; counts[blockIdx.x] = c; }
    return;
  }
  const uint64_t* nk = keys + lo;
  int32_t* dp = scratch + p.scratch_off + lo;
  const bool upd = p.slot >= 0;
  // ---- A: which new positions the existing list already holds; exclusive prefix of those duplicates -> dp --------------
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n_new; base += MT) {
    const int i = base + tid;
    int dup = 0;
    if (i < n_new && p.ex_n > 0) {
      const int32_t pos = (int32_t)(uint32_t)nk[i];
      const int k = lower_bound_i32(p.ex_pos, p.ex_n, pos);
      dup = k < p.ex_n && p.ex_pos[k] == pos;
    }
    int ex, total;
    Scan(tmp.scan).ExclusiveSum(dup, ex, total);
    if (i < n_new) dp[i] = carry + ex;
    __syncthreads();
    if (tid == 0) carry += total;
    __syncthreads();
  }
  if (tid == 0) dp[n_new] = carry;
  __syncthreads();
  const int n_dup = carry;
  // ---- B: the new entries (they win on equal positions) ----------------------------------------------------------------
  long long new_nulls = 0, union_nulls = 0, max_null = -1;
  unsigned long long vmin = ~0ull, vmax = 0;
  for (int i = tid; i < n_new; i += MT) {
    const int32_t pos = (int32_t)(uint32_t)nk[i];
    const int out = i + (p.ex_n > 0 ? lower_bound_i32(p.ex_pos, p.ex_n, pos) : 0) - dp[i];
    bool isnull = false;
    uint64_t raw = 0;
    if (upd) {
      const uint64_t* r = recs + (size_t)order[lo + i] * rec_words;
      isnull = (r[1] >> p.slot) & 1u;
      if (!isnull) {
        const uint64_t k = value_key(p.type, r[2 + p.slot]);
        vmin = min(vmin, (unsigned long long)k);
        vmax = max(vmax, (unsigned long long)k);
        raw = stored_bits(p.type, r[2 + p.slot]);
      }
      if (isnull) { new_nulls++; union_nulls++; max_null = max(max_null, (long long)out); }
    }
    if (WRITE) {
      p.out_pos[out] = pos;
      if (upd) { p.tmp_val[out] = raw; p.tmp_null[out] = isnull ? 1 : 0; }
    }
  }
  // ---- C: the existing entries the statement did not overwrite ---------------------------------------------------------
  __syncthreads();   // every thread has read n_dup out of `carry`
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < p.ex_n; base += MT) {
    const int j = base + tid;
    int isnull = 0;
    if (j < p.ex_n && upd && p.ex_nulls && (j >> 6) < p.ex_nwords) isnull = (int)((p.ex_nulls[j >> 6] >> (j & 63)) & 1ull);
    int nulls_before, total;
    Scan(tmp.scan).ExclusiveSum(isnull, nulls_before, total);
    if (j < p.ex_n) {
      const int32_t pos = p.ex_pos[j];
      const int k = lower_bound_key(nk, n_new, (uint32_t)pos);
      if (!(k < n_new && (int32_t)(uint32_t)nk[k] == pos)) {
        const int out = j + k - dp[k];
        if (upd && isnull) { union_nulls++; max_null = max(max_null, (long long)out); }
        if (WRITE) {
          p.out_pos[out] = pos;
          if (upd) { p.tmp_null[out] = (uint8_t)isnull; p.tmp_val[out] = isnull ? 0 : existing_bits(p, j - (carry + nulls_before)); }
        }
      }
    }
    __syncthreads();
    if (tid == 0) carry += total;
    __syncthreads();
  }
  const int n_union = n_new + p.ex_n - n_dup;
  if (!WRITE) {
    const long long s_new = RedI(tmp.ri).Sum(new_nulls);
    __syncthreads();
    const long long s_union = RedI(tmp.ri).Sum(union_nulls);
    __syncthreads();
    const long long m_null = RedI(tmp.ri).Reduce(max_null, cub::Max());
    __syncthreads();
    const unsigned long long mn = RedU(tmp.ru).Reduce(vmin, cub::Min());
    __syncthreads();
    const unsigned long long mx = RedU(tmp.ru).Reduce(vmax, cub::Max());
    if (tid == 0) {
      PairCounts c = {};
      c.n_new = n_new; c.n_union = n_union; c.union_nulls = s_union; c.new_nulls = s_new; c.max_null_idx = m_null;
      c.new_min = mn; c.new_max = mx;
      counts[blockIdx.x] = c;
    }
    return;
  }
  if (!upd) return;
  __syncthreads();   // tmp_null / tmp_val of the whole union are written
  // ---- D: null words (trimmed like the encoder does) and the non-null values, compacted in order -----------------------
  const int nwords = counts[blockIdx.x].max_null_idx >= 0 ? (int)(counts[blockIdx.x].max_null_idx / 64) + 1 : 0;
  for (int w = tid; w < nwords; w += MT) {
    uint64_t word = 0;
    for (int b = 0; b < 64; b++) { const int e = w * 64 + b; if (e < n_union && p.tmp_null[e]) word |= 1ull << b; }
    p.out_nulls[w] = word;
  }
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n_union; base += MT) {
    const int e = base + tid;
    const int nn = e < n_union && !p.tmp_null[e] ? 1 : 0;
    int vi, total;
    Scan(tmp.scan).ExclusiveSum(nn, vi, total);
    if (nn) {
      const uint64_t v = p.tmp_val[e];
      uint8_t* q = p.out_vals + (size_t)(carry + vi) * p.width;
      for (int k = 0; k < p.width; k++) q[k] = (uint8_t)(v >> (8 * k));
    }
    __syncthreads();
    if (tid == 0) carry += total;
    __syncthreads();
  }
}

__global__ void extract_keys(const uint64_t* recs, int rec_words, int64_t n, uint64_t* keys, uint32_t* idx) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    keys[i] = recs[(size_t)i * rec_words];
    idx[i] = (uint32_t)i;
  }
}
// [first, end) of every batch's records in the sorted order (seg is zeroed: batches without records stay empty)
__global__ void batch_segments(const uint64_t* keys, int64_t n, int32_t* seg) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t b = (uint32_t)(keys[i] >> 32);
    if (i == 0 || (uint32_t)(keys[i - 1] >> 32) != b) seg[2 * b] = (int32_t)i;
    if (i == n - 1 || (uint32_t)(keys[i + 1] >> 32) != b) seg[2 * b + 1] = (int32_t)(i + 1);
  }
}

int width_of_type(int t) {
  switch (t) {
    case SD_BYTE: return 1;
    case SD_SHORT: return 2;
    case SD_INT: case SD_DATE: case SD_FLOAT: return 4;
    case SD_LONG: case SD_TIMESTAMP: case SD_DOUBLE: case SD_DECIMAL: return 8;
  }
  return 0;
}

// ---- ColumnDelta.mergeStats (ColumnDelta.scala:134-222) on the host copy of a batch's stats row --------------------------
uint64_t key_to_raw(int type, uint64_t k) {   // inverse of value_key
  if (type != SD_FLOAT && type != SD_DOUBLE) return k ^ 0x8000000000000000ull;
  return (k >> 63) ? (k & 0x7fffffffffffffffull) : ~k;
}
// value of a stats slot as a sortable key (same order as value_key)
uint64_t slot_key(int type, const uint8_t* slot) {
  uint64_t raw = 0;
  switch (type) {
    case SD_BYTE: { int8_t v; memcpy(&v, slot, 1); raw = (uint64_t)(int64_t)v; break; }
    case SD_SHORT: { int16_t v; memcpy(&v, slot, 2); raw = (uint64_t)(int64_t)v; break; }
    case SD_INT: case SD_DATE: { int32_t v; memcpy(&v, slot, 4); raw = (uint64_t)(int64_t)v; break; }
    case SD_FLOAT: { float f; memcpy(&f, slot, 4); double d = f; memcpy(&raw, &d, 8); break; }
    default: memcpy(&raw, slot, 8);
  }
  if (type != SD_FLOAT && type != SD_DOUBLE) return raw ^ 0x8000000000000000ull;
  double d; memcpy(&d, &raw, 8);
  if (d != d) raw = 0x7ff8000000000000ull;
  return (raw >> 63) ? ~raw : (raw | 0x8000000000000000ull);
}
void write_slot(int type, uint8_t* slot, uint64_t key) {
  const uint64_t raw = key_to_raw(type, key);
  memset(slot, 0, 8);
  switch (type) {
    case SD_BYTE: { int8_t v = (int8_t)(int64_t)raw; memcpy(slot, &v, 1); break; }
    case SD_SHORT: { int16_t v = (int16_t)(int64_t)raw; memcpy(slot, &v, 2); break; }
    case SD_INT: case SD_DATE: { int32_t v = (int32_t)(int64_t)raw; memcpy(slot, &v, 4); break; }
    case SD_FLOAT: { double d; memcpy(&d, &raw, 8); float f = (float)d; memcpy(slot, &f, 4); break; }
    default: memcpy(slot, &raw, 8);
  }
}
void merge_stats(std::vector<uint8_t>& row, int stats_ncols, int table_col, int type, const PairCounts& c) {
  const int nf = 1 + 3 * stats_ncols;
  const size_t bits = (size_t)((nf + 63) / 64) * 8;
  if (row.size() < bits + 8 * (size_t)nf) return;
  auto isnull = [&](int f) { return (row[(size_t)f >> 3] >> (f & 7)) & 1; };
  auto slot = [&](int f) { return row.data() + bits + 8 * (size_t)f; };
  int32_t count;
  memcpy(&count, slot(0), 4);
  count = -std::abs(count);   // negative batch count: the batch has update deltas
  memcpy(slot(0), &count, 4);
  if (table_col >= stats_ncols) return;
  const int flo = 1 + 3 * table_col, fhi = flo + 1, fnc = flo + 2;
  if (c.n_new > c.new_nulls) {   // lower / upper widen by the new non-null values (a NULL bound takes the new one)
    if (isnull(flo) || c.new_min < slot_key(type, slot(flo))) { write_slot(type, slot(flo), c.new_min); row[(size_t)flo >> 3] &= (uint8_t)~(1u << (flo & 7)); }
    if (isnull(fhi) || slot_key(type, slot(fhi)) < c.new_max) { write_slot(type, slot(fhi), c.new_max); row[(size_t)fhi >> 3] &= (uint8_t)~(1u << (fhi & 7)); }
  }
  int32_t old_nc;
  memcpy(&old_nc, slot(fnc), 4);
  int64_t nc = std::max<int64_t>((int64_t)old_nc - (c.n_new - c.new_nulls), c.new_nulls);
  if (nc <= 0 && old_nc > 0) nc = 1;
  const int32_t v = (int32_t)nc;
  memcpy(slot(fnc), &v, 4);
}

struct Timing { double scan_ms = 0, sort_ms = 0, merge_ms = 0, install_ms = 0, total_ms = 0, rows = 0; };
thread_local Timing g_timing;

int run_statement(sd_plan* p, sd_store* s, const int32_t* bucket_ids, int32_t nbuckets, const sd_literal* lits, int32_t nlits,
                  const int32_t* target_cols, int64_t* rows_out, const char* what) {
  const auto t0 = std::chrono::steady_clock::now();
  if (!p || !s || !rows_out) return set_error(SD_ERR_INVALID, "%s: null argument", what);
  const PlanSpec& sp = plan_spec(p);
  if (sp.mode != MODE_MUTATE) return set_error(SD_ERR_STATE, "%s: the plan is not an UPDATE / DELETE plan (sd_plan_desc.flags lacks SD_PLAN_MUTATE)", what);
  const bool upd = target_cols != nullptr;
  const int T = upd ? (int)sp.proj.size() : 1;
  if (upd && T == 0) return set_error(SD_ERR_INVALID, "%s: an UPDATE plan needs one SET value per target", what);
  if (!upd && !sp.proj.empty()) return set_error(SD_ERR_INVALID, "%s: a DELETE plan has no SET values (nproj = 0)", what);
  std::vector<int> tcol(T, -1), ttype(T, 0), twidth(T, 0), tnullable(T, 0);
  for (int t = 0; upd && t < T; t++) {
    const int c = target_cols[t];
    if (c < 0 || c >= (int)s->schema.size()) return set_error(SD_ERR_INVALID, "%s: target column %d outside the store schema", what, c);
    for (int u = 0; u < t; u++) if (tcol[u] == c) return set_error(SD_ERR_INVALID, "%s: table column %d is assigned twice", what, c);
    const sd_column& sc = s->schema[c];
    if (sc.type == SD_STRING || sc.type == SD_BOOLEAN)
      return set_error(SD_ERR_UNSUPPORTED, "%s: STRING / BOOLEAN targets (Dictionary / BooleanBitSet delta encoders) are not executed on the device", what);
    const sd_expr& e = sp.exprs[sp.proj[t]];
    if (e.type != sc.type) return set_error(SD_ERR_INVALID, "%s: SET value %d has sd_type %d, target column %d is %d", what, t, e.type, c, sc.type);
    if (sc.type == SD_DECIMAL && decimal_ps(sp, sp.proj[t]) != SD_DEC_PS(sc.precision, sc.scale))
      return set_error(SD_ERR_INVALID, "%s: SET value %d is not DECIMAL(%d,%d) like target column %d", what, t, sc.precision, sc.scale, c);
    tcol[t] = c; ttype[t] = sc.type; twidth[t] = width_of_type(sc.type); tnullable[t] = sc.nullable;
  }
  std::lock_guard<std::mutex> serial(s->mutate_mu);   // statements on one store run one after the other
  MutationScan ms;
  int rc = mutation_scan(p, s, bucket_ids, nbuckets, lits, nlits, &ms);
  if (rc) return rc;
  g_timing = Timing();
  g_timing.scan_ms = ms.scan_ms;
  *rows_out = 0;
  if (ms.count == 0) return 0;
  if (ms.count >= INT32_MAX) return set_error(SD_ERR_UNSUPPORTED, "%s: more than 2^31 rows in one statement", what);
  const int nb = (int)ms.batches.size();
  const int n = (int)ms.count;
  cudaStream_t st = ms.stream;
  cudaEvent_t ev[3];
  for (auto& e : ev) SD_CUDA(cudaEventCreate(&e));
  struct EvGuard { cudaEvent_t* e; ~EvGuard() { for (int i = 0; i < 3; i++) cudaEventDestroy(e[i]); } } evg{ev};
  DevScratch ds;
  ds.st = st;
  // ---- sort the records by (batch, row) --------------------------------------------------------------------------------
  uint64_t *k_in, *k_out;
  uint32_t *i_in, *i_out;
  int32_t* d_seg;
  if ((rc = ds.get(&k_in, 8 * (size_t)n)) || (rc = ds.get(&k_out, 8 * (size_t)n)) || (rc = ds.get(&i_in, 4 * (size_t)n)) ||
      (rc = ds.get(&i_out, 4 * (size_t)n)) || (rc = ds.get(&d_seg, 8 * (size_t)nb)))
    return rc;
  SD_CUDA(cudaEventRecord(ev[0], st));
  const int grid = (int)std::min<int64_t>(4096, (n + 255) / 256);
  extract_keys<<<grid, 256, 0, st>>>(ms.records, ms.rec_words, n, k_in, i_in);
  int end_bit = 32;
  while (end_bit < 64 && (1ll << (end_bit - 32)) < nb) end_bit++;
  size_t tb = 0;
  SD_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, k_in, k_out, i_in, i_out, n, 0, end_bit, st));
  void* d_tmp = nullptr;
  if ((rc = ds.get(&d_tmp, tb))) return rc;
  SD_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp, tb, k_in, k_out, i_in, i_out, n, 0, end_bit, st));
  SD_CUDA(cudaMemsetAsync(d_seg, 0, 8 * (size_t)nb, st));
  batch_segments<<<grid, 256, 0, st>>>(k_out, n, d_seg);
  SD_CUDA(cudaGetLastError());
  SD_CUDA(cudaEventRecord(ev[1], st));
  // ---- pairs + counting pass -------------------------------------------------------------------------------------------
  std::vector<MergePair> pairs((size_t)nb * T);
  std::vector<std::string> problem((size_t)nb * T);   // reported only when the pair turns out to be touched
  std::vector<int> problem_code((size_t)nb * T, SD_ERR_UNSUPPORTED);
  for (int b = 0; b < nb; b++) {
    const StoredBatch& sb = *ms.batches[b];
    for (int t = 0; t < T; t++) {
      MergePair& mp = pairs[(size_t)b * T + t];
      memset(&mp, 0, sizeof(mp));
      mp.batch = b; mp.slot = upd ? t : -1; mp.type = ttype[t]; mp.width = twidth[t];
      mp.scratch_off = (int64_t)t * (n + nb) + b;   // 64-bit: T * (n + nb) may pass 2^31
      if (!upd) {
        mp.ex_pos = sb.dev_deletes; mp.ex_n = sb.num_deletes;
        continue;
      }
      const int c = tcol[t];
      if (c >= (int)sb.cols.size() || !sb.cols[c].present) { problem[(size_t)b * T + t] = "target column not resident"; problem_code[(size_t)b * T + t] = SD_ERR_INVALID; continue; }
      const StoredCol& col = sb.cols[c];
      if (!col.unsupported.empty()) { problem[(size_t)b * T + t] = col.unsupported; continue; }
      const StoredDelta& d = col.delta[0];
      if (!d.present) continue;
      const bool dict_ok = (d.dev.enc == ENC_DICTIONARY || d.dev.enc == ENC_BIG_DICTIONARY) && d.dev.dict &&
                           (ttype[t] == SD_INT || ttype[t] == SD_DATE || ttype[t] == SD_LONG || ttype[t] == SD_TIMESTAMP);
      if (d.dev.enc != ENC_UNCOMPRESSED && !dict_ok) { problem[(size_t)b * T + t] = "existing depth-0 delta in an encoding the merge does not read"; continue; }
      mp.ex_pos = d.dev.positions; mp.ex_n = d.dev.n; mp.ex_nulls = d.dev.nulls; mp.ex_nwords = d.dev.nwords;
      mp.ex_data = d.dev.data; mp.ex_dict = d.dev.dict; mp.ex_enc = d.dev.enc;
    }
  }
  // scratch of the duplicate prefixes: pair (b, t) uses [t * (n + nb) + first record of b + b, ... + n_new + 1)
  int32_t* d_scratch;
  MergePair* d_pairs;
  PairCounts* d_counts;
  if ((rc = ds.get(&d_scratch, 4 * (size_t)T * ((size_t)n + nb))) || (rc = ds.get(&d_pairs, sizeof(MergePair) * pairs.size())) ||
      (rc = ds.get(&d_counts, sizeof(PairCounts) * pairs.size())))
    return rc;
  SD_CUDA(cudaMemcpyAsync(d_pairs, pairs.data(), sizeof(MergePair) * pairs.size(), cudaMemcpyHostToDevice, st));
  merge_kernel<false><<<(int)pairs.size(), MT, 0, st>>>(d_pairs, k_out, i_out, ms.records, ms.rec_words, d_seg, d_scratch, d_counts);
  SD_CUDA(cudaGetLastError());
  std::vector<PairCounts> counts(pairs.size());
  SD_CUDA(cudaMemcpyAsync(counts.data(), d_counts, sizeof(PairCounts) * counts.size(), cudaMemcpyDeviceToHost, st));
  SD_CUDA(cudaStreamSynchronize(st));
  for (size_t i = 0; i < pairs.size(); i++) {
    if (counts[i].n_new == 0) continue;
    if (!problem[i].empty()) return set_error(problem_code[i], "%s: batch %lld column %d: %s", what,
                                              (long long)ms.batches[pairs[i].batch]->batch_id, tcol[i % T], problem[i].c_str());
    if (upd && counts[i].new_nulls > 0 && !tnullable[i % T])
      return set_error(SD_ERR_INVALID, "%s: NULL assigned to NOT NULL column %d", what, tcol[i % T]);
  }
  // ---- layout in the store's arena, all outputs of the statement at once -----------------------------------------------
  size_t tmp_entries = 0;
  for (size_t i = 0; i < pairs.size(); i++) if (counts[i].n_new) tmp_entries += (size_t)counts[i].n_union;
  uint64_t* d_tval = nullptr;
  uint8_t* d_tnull = nullptr;
  if (upd && ((rc = ds.get(&d_tval, 8 * tmp_entries)) || (rc = ds.get(&d_tnull, tmp_entries)))) return rc;
  std::vector<DevDelta> devd(pairs.size());
  DevDelta* d_devd = nullptr;
  std::vector<std::vector<Extent>> new_extents(nb);   // per batch: the allocations its new version adds
  {
    std::lock_guard<std::mutex> lock(s->mu);
    size_t toff = 0;
    for (size_t i = 0; i < pairs.size(); i++) {
      const PairCounts& c = counts[i];
      if (!c.n_new) continue;
      ExtentRecorder rec(s->arena, &new_extents[i / T]);
      MergePair& mp = pairs[i];
      mp.out_pos = reinterpret_cast<int32_t*>(s->arena.alloc(4 * (size_t)c.n_union + 16, 16));
      if (!mp.out_pos) return SD_ERR_CUDA;
      if (!upd) continue;
      const int nw = c.max_null_idx >= 0 ? (int)(c.max_null_idx / 64) + 1 : 0;
      if (nw) { mp.out_nulls = reinterpret_cast<uint64_t*>(s->arena.alloc(8 * (size_t)nw, 8)); if (!mp.out_nulls) return SD_ERR_CUDA; }
      mp.out_vals = s->arena.alloc((size_t)(c.n_union - c.union_nulls) * mp.width + 160, 16);   // tail padding like upload_bytes
      if (!mp.out_vals) return SD_ERR_CUDA;
      mp.tmp_val = d_tval + toff; mp.tmp_null = d_tnull + toff;
      toff += (size_t)c.n_union;
      DevDelta& dd = devd[i];
      memset(&dd, 0, sizeof(dd));
      dd.positions = mp.out_pos; dd.data = mp.out_vals; dd.nulls = nw ? mp.out_nulls : nullptr;
      dd.n = (int32_t)c.n_union; dd.nwords = nw; dd.enc = ENC_UNCOMPRESSED;
    }
    if (upd) {
      d_devd = reinterpret_cast<DevDelta*>(s->arena.alloc(sizeof(DevDelta) * devd.size(), 16));
      if (!d_devd) return SD_ERR_CUDA;
      for (int b = 0; b < nb; b++)   // each batch owns its slice of the statement's DevDelta array
        if (!new_extents[b].empty()) new_extents[b].push_back(Extent{reinterpret_cast<uint8_t*>(d_devd + (size_t)b * T), sizeof(DevDelta) * T});
    }
  }
  // ---- writing pass ----------------------------------------------------------------------------------------------------
  SD_CUDA(cudaMemcpyAsync(d_pairs, pairs.data(), sizeof(MergePair) * pairs.size(), cudaMemcpyHostToDevice, st));
  merge_kernel<true><<<(int)pairs.size(), MT, 0, st>>>(d_pairs, k_out, i_out, ms.records, ms.rec_words, d_seg, d_scratch, d_counts);
  SD_CUDA(cudaGetLastError());
  if (upd) SD_CUDA(cudaMemcpyAsync(d_devd, devd.data(), sizeof(DevDelta) * devd.size(), cudaMemcpyHostToDevice, st));
  SD_CUDA(cudaEventRecord(ev[2], st));
  SD_CUDA(cudaStreamSynchronize(st));
  const auto t_inst = std::chrono::steady_clock::now();
  // ---- new batch versions -------------------------------------------------------------------------------------------------
  FreshBatches fresh;
  for (int b = 0; b < nb; b++) {
    bool touched = false;
    for (int t = 0; t < T; t++) touched = touched || counts[(size_t)b * T + t].n_new > 0;
    if (!touched) continue;
    const StoredBatch& old = *ms.batches[b];
    std::unique_ptr<StoredBatch> nbp(new StoredBatch(old));
    nbp->uid = next_batch_uid();
    nbp->extents.insert(nbp->extents.end(), new_extents[b].begin(), new_extents[b].end());   // (replaced ones pruned at install)
    for (int t = 0; t < T; t++) {
      const size_t i = (size_t)b * T + t;
      const PairCounts& c = counts[i];
      if (!upd) {
        nbp->dev_deletes = pairs[i].out_pos;
        nbp->num_deletes = (int32_t)c.n_union;
        nbp->gone = c.n_union >= old.num_rows;   // ColumnDelta.checkBatchDeleted
        continue;
      }
      StoredCol& col = nbp->cols[tcol[t]];
      StoredDelta nd;
      nd.present = true;
      nd.dev = devd[i];
      nd.nbase = old.num_rows;
      nd.body_off = ((8 + 8 * (int64_t)devd[i].nwords + 8 + 4 * c.n_union + 7) >> 3) << 3;
      nd.len = nd.body_off + (c.n_union - c.union_nulls) * pairs[i].width;
      col.delta[0] = nd;
      col.dev_delta[0] = d_devd + i;
      col.dev.delta0 = d_devd + i;
      col.fast = false;
      nbp->has_deltas = true;
      if (!nbp->stats.empty()) merge_stats(nbp->stats, nbp->stats_ncols, tcol[t], ttype[t], c);
    }
    fresh.emplace_back(&old, std::move(nbp));
  }
  // install: every new version of the statement under one hold of the store's lock
  if ((rc = store_install(s, fresh, {}, what))) return rc;
  *rows_out = ms.count;
  const auto t1 = std::chrono::steady_clock::now();
  float a = 0, bms = 0;
  cudaEventElapsedTime(&a, ev[0], ev[1]);
  cudaEventElapsedTime(&bms, ev[1], ev[2]);
  g_timing.sort_ms = a;
  g_timing.merge_ms = bms;
  g_timing.install_ms = std::chrono::duration<double, std::milli>(t1 - t_inst).count();
  g_timing.total_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
  g_timing.rows = (double)ms.count;
  return 0;
}

}  // namespace
}  // namespace sd

extern "C" {

int sd_plan_update_store(sd_plan* p, sd_store* s, const int32_t* bucket_ids, int32_t nbuckets, const sd_literal* lits, int32_t nlits,
                         const int32_t* target_cols, int64_t* rows_updated) {
  if (!target_cols) return sd::set_error(SD_ERR_INVALID, "sd_plan_update_store: null target_cols");
  return sd::run_statement(p, s, bucket_ids, nbuckets, lits, nlits, target_cols, rows_updated, "sd_plan_update_store");
}

int sd_plan_delete_store(sd_plan* p, sd_store* s, const int32_t* bucket_ids, int32_t nbuckets, const sd_literal* lits, int32_t nlits,
                         int64_t* rows_deleted) {
  return sd::run_statement(p, s, bucket_ids, nbuckets, lits, nlits, nullptr, rows_deleted, "sd_plan_delete_store");
}

// host clock and device times of the calling thread's last UPDATE / DELETE (tools/mutation_bench.py):
// [0] scan kernels ms [1] sort ms [2] count + write merge ms [3] host install ms [4] whole statement ms [5] rows
int sdx_last_mutation_timing(double out[6]) {
  const sd::Timing& t = sd::g_timing;
  out[0] = t.scan_ms; out[1] = t.sort_ms; out[2] = t.merge_ms; out[3] = t.install_ms; out[4] = t.total_ms; out[5] = t.rows;
  return 0;
}

int sdx_store_get_delta(sd_store* s, int64_t batch_index, int32_t table_col, int32_t depth, void* out, int64_t cap, int64_t* out_len) {
  if (!s || !out_len) return sd::set_error(SD_ERR_INVALID, "sdx_store_get_delta: null argument");
  if (depth != 0 && depth != 1) return sd::set_error(SD_ERR_INVALID, "sdx_store_get_delta: depth %d", depth);
  std::lock_guard<std::mutex> lock(s->mu);
  if (batch_index < 0 || batch_index >= (int64_t)s->batches.size()) return sd::set_error(SD_ERR_INVALID, "batch index out of range");
  const sd::StoredBatch& b = *s->batches[batch_index];
  if (table_col < 0 || table_col >= (int)b.cols.size() || !b.cols[table_col].present || !b.cols[table_col].delta[depth].present)
    return sd::set_error(SD_ERR_INVALID, "column %d has no depth-%d delta", table_col, depth);
  const sd::StoredDelta& d = b.cols[table_col].delta[depth];
  if (d.dev.enc != sd::ENC_UNCOMPRESSED) return sd::set_error(SD_ERR_UNSUPPORTED, "sdx_store_get_delta: only Uncompressed deltas are rebuilt");
  *out_len = d.len;
  if (cap < d.len) return sd::set_error(SD_ERR_OVERFLOW, "buffer too small");
  SD_CUDA(cudaSetDevice(s->device));
  uint8_t* o = reinterpret_cast<uint8_t*>(out);
  memset(o, 0, (size_t)d.len);
  const int32_t hdr[2] = {d.dev.enc, 8 * d.dev.nwords};
  memcpy(o, hdr, 8);
  if (d.dev.nwords) SD_CUDA(cudaMemcpy(o + 8, d.dev.nulls, 8 * (size_t)d.dev.nwords, cudaMemcpyDeviceToHost));
  uint8_t* q = o + 8 + 8 * (size_t)d.dev.nwords;
  const int32_t mid[2] = {d.nbase, d.dev.n};
  memcpy(q, mid, 8);
  if (d.dev.n) SD_CUDA(cudaMemcpy(q + 8, d.dev.positions, 4 * (size_t)d.dev.n, cudaMemcpyDeviceToHost));
  if (d.len > d.body_off) SD_CUDA(cudaMemcpy(o + d.body_off, d.dev.data, (size_t)(d.len - d.body_off), cudaMemcpyDeviceToHost));
  return 0;
}

int sdx_store_get_deletes(sd_store* s, int64_t batch_index, void* out, int64_t cap, int64_t* out_len) {
  if (!s || !out_len) return sd::set_error(SD_ERR_INVALID, "sdx_store_get_deletes: null argument");
  std::lock_guard<std::mutex> lock(s->mu);
  if (batch_index < 0 || batch_index >= (int64_t)s->batches.size()) return sd::set_error(SD_ERR_INVALID, "batch index out of range");
  const sd::StoredBatch& b = *s->batches[batch_index];
  if (!b.dev_deletes) return sd::set_error(SD_ERR_INVALID, "batch %lld has no delete mask", (long long)batch_index);
  *out_len = 12 + 4 * (int64_t)b.num_deletes;
  if (cap < *out_len) return sd::set_error(SD_ERR_OVERFLOW, "buffer too small");
  SD_CUDA(cudaSetDevice(s->device));
  const int32_t hdr[3] = {0, b.num_rows, b.num_deletes};
  memcpy(out, hdr, 12);
  if (b.num_deletes) SD_CUDA(cudaMemcpy(reinterpret_cast<uint8_t*>(out) + 12, b.dev_deletes, 4 * (size_t)b.num_deletes, cudaMemcpyDeviceToHost));
  return 0;
}

}  // extern "C"
