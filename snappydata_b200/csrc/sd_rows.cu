// MODE_PROJECT: the projection records of an execution -> UnsafeRows, ON THE DEVICE.
//
// The scan kernel leaves one fixed-width record per passing row ([batch ordinal | null bits][8 bytes per projected field], string
// fields as dictionary codes or positions of the value's [len][bytes] record).  Round 1 / early round 2 read the records back
// and built the rows in a host loop (dictionary lookups that miss the cache, a serial writer), which took most of a C4
// step.  Here the rows are sized, laid out (exclusive scan) and written
// by the GPU, where the dictionaries already are, and leave in ONE copy straight into the caller's buffer.
//
// Row format (what ColumnTableScan's generated code appends to its output buffer, and what
// snappydata_b200.column_format.parse_row_stream / the oracle's emit_unsafe_row produce):
//   [int64 size][null-bit words][8-byte slot per field][variable part: string bytes, each padded to 8]
//   string slot = (offset from the start of the null words << 32) | length; narrow fields in the low bytes of their slot.
#include <cub/device/device_scan.cuh>

#include "sd_host.h"

namespace sd {

namespace {

struct RowWriteParams {
  const uint64_t* recs;
  int64_t count;
  int32_t np, nstr, nbatches, fixed;   // fixed = null words + slots, bytes
  uint8_t kind[ROW_MAX_FIELDS];
  int8_t sidx[ROW_MAX_FIELDS];         // field -> index among the string fields
  const RowStrSrc* src;                // [nbatches][nstr]
  int64_t* offs;                       // sizes, then (in place) offsets; [count + 1]
  uint8_t* out;
  int32_t* err;
};

__device__ __forceinline__ int32_t load_i32_unaligned(const uint8_t* p) {
  return (int32_t)((uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24));
}

// the value of string field j of a record: its bytes and length; NULL when the code is the column's NULL code
__device__ __forceinline__ int32_t string_of(const RowWriteParams& P, uint32_t bidx, int j, uint64_t raw, const uint8_t*& bytes, bool& isnull) {
  const RowStrSrc s = P.src[(size_t)bidx * (size_t)P.nstr + (size_t)P.sidx[j]];
  const uint8_t* rec;
  if (!s.rec_off) {
    rec = s.base + (uint32_t)raw;
  } else {
    const int64_t code = (int64_t)raw;
    if (code == (int64_t)s.null_code && code >= 0) { isnull = true; return 0; }
    if (code < 0 || code >= (int64_t)s.n) { atomicExch(P.err, 2); isnull = true; return 0; }
    rec = s.base + s.rec_off[code];
  }
  const int32_t len = load_i32_unaligned(rec);
  if (len < 0) { atomicExch(P.err, 3); isnull = true; return 0; }
  bytes = rec + 4;
  return len;
}

__global__ void __launch_bounds__(256) row_sizes_kernel(const RowWriteParams P) {
  const int rw = 1 + P.np;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= P.count; i += (int64_t)gridDim.x * blockDim.x) {
    if (i == P.count) { P.offs[i] = 0; continue; }
    const uint64_t* r = P.recs + (size_t)i * (size_t)rw;
    const uint32_t bidx = (uint32_t)(r[0] & 0xffffffffu), pnull = (uint32_t)(r[0] >> 32);
    int64_t var = 0;
    if (bidx >= (uint32_t)P.nbatches) { atomicExch(P.err, 1); P.offs[i] = 8 + P.fixed; continue; }
    for (int j = 0; j < P.np; j++) {
      if (P.kind[j] != ROW_KIND_STRING || ((pnull >> j) & 1u)) continue;
      const uint8_t* b = nullptr;
      bool isnull = false;
      const int32_t len = string_of(P, bidx, j, r[1 + j], b, isnull);
      var += ((int64_t)len + 7) & ~int64_t(7);
    }
    P.offs[i] = 8 + (int64_t)P.fixed + var;
  }
}

// one warp per row: lane j owns field j (np <= 32)
__global__ void __launch_bounds__(256) row_write_kernel(const RowWriteParams P) {
  const int lane = threadIdx.x & 31;
  const int rw = 1 + P.np;
  const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = warp0; i < P.count; i += nwarps) {
    const uint64_t* r = P.recs + (size_t)i * (size_t)rw;
    const uint64_t head = r[0];
    const uint32_t bidx = (uint32_t)(head & 0xffffffffu), pnull = (uint32_t)(head >> 32);
    if (bidx >= (uint32_t)P.nbatches) continue;   // (flagged by the size pass)
    const bool mine = lane < P.np;
    const int kind = mine ? P.kind[lane] : 0;
    const uint64_t raw = mine ? r[1 + lane] : 0ull;
    bool isnull = mine && ((pnull >> lane) & 1u);
    const uint8_t* bytes = nullptr;
    int32_t len = 0;
    if (mine && !isnull && kind == ROW_KIND_STRING) len = string_of(P, bidx, lane, raw, bytes, isnull);
    const int32_t pad = (len + 7) & ~7;
    int32_t incl = pad;   // inclusive scan of the padded lengths: where each string starts in the variable part
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int32_t o = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += o;
    }
    const int32_t voff = P.fixed + incl - pad;
    uint64_t slot = 0;
    if (mine && !isnull) {
      switch (kind) {
        case ROW_KIND_BOOL: slot = raw != 0ull; break;
        case ROW_KIND_1: slot = raw & 0xffull; break;
        case ROW_KIND_2: slot = raw & 0xffffull; break;
        case ROW_KIND_4: slot = raw & 0xffffffffull; break;
        case ROW_KIND_FLOAT: slot = (uint64_t)__float_as_uint((float)__longlong_as_double((long long)raw)); break;
        case ROW_KIND_STRING: slot = ((uint64_t)(uint32_t)voff << 32) | (uint64_t)(uint32_t)len; break;
        default: slot = raw; break;
      }
    }
    const uint32_t nullmask = __ballot_sync(0xffffffffu, isnull);
    const int64_t o0 = P.offs[i];
    uint8_t* row = P.out + o0;
    if (lane == 0) {
      *reinterpret_cast<int64_t*>(row) = P.offs[i + 1] - o0 - 8;
      *reinterpret_cast<uint64_t*>(row + 8) = (uint64_t)nullmask;
    }
    const int bits = P.fixed - 8 * P.np;
    if (mine) *reinterpret_cast<uint64_t*>(row + 8 + bits + 8 * lane) = slot;
    uint32_t smask = __ballot_sync(0xffffffffu, len > 0);
    while (smask) {   // every string of the row, copied by the whole warp (the padding is already zero)
      const int L = __ffs(smask) - 1;
      smask &= smask - 1u;
      const uint8_t* b = reinterpret_cast<const uint8_t*>(__shfl_sync(0xffffffffu, (unsigned long long)(uintptr_t)bytes, L));
      const int32_t l = __shfl_sync(0xffffffffu, len, L);
      const int32_t d = __shfl_sync(0xffffffffu, voff, L);
      for (int32_t k = lane; k < l; k += 32) row[8 + d + k] = b[k];
    }
  }
}

template <typename T>
int grow(T*& p, size_t& cap, size_t need) {
  if (need <= cap) return 0;
  if (p) cudaFree(p);
  p = nullptr; cap = 0;
  const size_t want = need + need / 4 + 4096;
  cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&p), want);
  if (e != cudaSuccess) return set_error(SD_ERR_CUDA, "cudaMalloc(%zu) for the projected rows: %s", want, cudaGetErrorString(e));
  cap = want;
  return 0;
}

}  // namespace

void RowWriterBuffers::release() {
  if (d_offs) cudaFree(d_offs);
  if (d_tmp) cudaFree(d_tmp);
  if (d_rows) cudaFree(d_rows);
  if (d_err) cudaFree(d_err);
  if (d_src) cudaFree(d_src);
  if (d_recoff) cudaFree(d_recoff);
  *this = RowWriterBuffers();
}

// records (device) -> rows (device, b.d_rows); *total_out = bytes of the row stream
int device_write_rows(cudaStream_t st, const uint64_t* d_recs, int64_t count, int np, const uint8_t* kinds, int nbatches,
                      RowWriterBuffers& b, int64_t* total_out) {
#define RW(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return set_error(SD_ERR_CUDA, "%s: %s", #call, cudaGetErrorString(e_)); } while (0)
  *total_out = 0;
  if (count <= 0) return 0;
  if (np > ROW_MAX_FIELDS) return set_error(SD_ERR_UNSUPPORTED, "device row writer: %d fields", np);
  RowWriteParams P = {};
  P.recs = d_recs; P.count = count; P.np = np; P.nbatches = nbatches;
  P.fixed = ((np + 63) / 64) * 8 + 8 * np;
  int ns = 0;
  for (int j = 0; j < np; j++) { P.kind[j] = kinds[j]; P.sidx[j] = kinds[j] == ROW_KIND_STRING ? (int8_t)ns++ : (int8_t)-1; }
  P.nstr = ns;
  P.src = b.d_src;
  int rc = grow(b.d_offs, b.offs_cap, ((size_t)count + 1) * 8);
  if (rc) return rc;
  if (!b.d_err) RW(cudaMalloc(reinterpret_cast<void**>(&b.d_err), 8));
  RW(cudaMemsetAsync(b.d_err, 0, 8, st));
  P.offs = b.d_offs; P.err = b.d_err;
  int dev = 0, sms = 0;
  RW(cudaGetDevice(&dev));
  RW(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int blocks = (int)std::min<int64_t>(sms * 8, (count + 256) / 256);
  row_sizes_kernel<<<blocks, 256, 0, st>>>(P);
  RW(cudaGetLastError());
  size_t tmp = 0;
  RW(cub::DeviceScan::ExclusiveSum(nullptr, tmp, b.d_offs, b.d_offs, (int)(count + 1), st));
  { uint8_t* t = reinterpret_cast<uint8_t*>(b.d_tmp); rc = grow(t, b.tmp_cap, tmp + 16); b.d_tmp = t; if (rc) return rc; }
  RW(cub::DeviceScan::ExclusiveSum(b.d_tmp, tmp, b.d_offs, b.d_offs, (int)(count + 1), st));
  int64_t total = 0;
  int32_t err = 0;
  RW(cudaMemcpyAsync(&total, b.d_offs + count, 8, cudaMemcpyDeviceToHost, st));
  RW(cudaMemcpyAsync(&err, b.d_err, 4, cudaMemcpyDeviceToHost, st));
  RW(cudaStreamSynchronize(st));
  if (err) return set_error(SD_ERR_CUDA, err == 1 ? "corrupt projection record (batch ordinal)" : err == 2 ? "dictionary code out of range in a projection record" : "corrupt string record");
  rc = grow(b.d_rows, b.rows_cap, (size_t)total + 64);
  if (rc) return rc;
  RW(cudaMemsetAsync(b.d_rows, 0, (size_t)total, st));
  P.out = b.d_rows;
  const int wblocks = (int)std::min<int64_t>(sms * 8, (count * 32 + 255) / 256);
  row_write_kernel<<<wblocks, 256, 0, st>>>(P);
  RW(cudaGetLastError());
  *total_out = total;
#undef RW
  return 0;
}

}  // namespace sd
