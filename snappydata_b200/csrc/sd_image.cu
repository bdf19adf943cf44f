// sd_image.cu -- scan images of resident columns: the same values in fewer bytes, for the staged loads of the scan kernel.
//
// A resident column's verbatim bytes stay the only source of truth (export, mutations, compaction and the per-row paths read
// them).  An image is a read-only copy that a batch version owns beside them, byte-aligned so that the kernel's bulk copies
// and conflict-free consumer loads keep their shape:
//   DOUBLE / FLOAT                   <= 256 distinct BIT PATTERNS in the batch: 1-byte indexes into a sorted table of them
//                                    (so -0.0 / +0.0 and NaN payloads stay distinct)
//   SHORT / INT / DATE / LONG /      max - min < 2^8 or 2^16: unsigned offsets from min in 1 or 2 bytes, when narrower
//   TIMESTAMP / dictionary codes     than the verbatim element
// Only NOT NULL-in-this-batch columns of batches of >= IMG_MIN_ROWS rows get one.  The build is two launches of one CTA per (batch, column): the first finds
// the distinct bit patterns (shared-memory open-addressing set) or the range, the host places the chosen images in the
// store's arena, the second writes them and then decodes every row back and compares it with the verbatim bytes.  A
// (batch, column) that does not match bit for bit keeps no image and counts in sd_store::image_mismatches.
#include "sd_host.h"

#include <chrono>
#include <climits>

namespace sd {

int image_width(bool dict, int ew, uint64_t ndistinct, int64_t lo, int64_t hi) {
  if (dict) return ndistinct <= (uint64_t)IMG_DICT_MAX ? 1 : 0;
  const uint64_t range = (uint64_t)hi - (uint64_t)lo;
  const int w = range <= 0xffull ? 1 : range <= 0xffffull ? 2 : 8;
  return w < ew ? w : 0;
}

namespace {

struct ImageJob {
  const uint8_t* src;     // verbatim values
  uint8_t* img;           // encode pass: where the codes go (img_tab = img - tab_bytes)
  uint64_t* tab;          // encode pass: the table in the arena
  int64_t n;
  int32_t ew;             // element bytes: 2, 4 or 8
  int32_t dict;           // 1: dictionary of bit patterns (floating point), 0: frame of reference (signed integers)
  // analysis results (the host picks the width from them)
  int32_t width;          // 0: no image
  int32_t ndict;          // distinct bit patterns; IMG_DICT_MAX + 1: more
  int64_t lo, hi;
  int64_t mismatches;     // encode pass: rows whose decoded image differs from the verbatim value
};

constexpr int IMG_THREADS = 256;
// smaller batches keep the verbatim path: their tile copies are a few 16-byte units either way, and the two host
// synchronisations of a build would cost more than the scan saves
constexpr int IMG_MIN_ROWS = 1024;
constexpr int SET_SLOTS = 2 * IMG_DICT_MAX;
constexpr uint64_t SET_EMPTY = ~0ull;

__device__ __forceinline__ uint64_t elem_bits(const uint8_t* p, int ew, int64_t i) {   // zero-extended bit pattern
  return ew == 8 ? reinterpret_cast<const uint64_t*>(p)[i] : ew == 4 ? (uint64_t)reinterpret_cast<const uint32_t*>(p)[i]
                                                                      : (uint64_t)reinterpret_cast<const uint16_t*>(p)[i];
}
__device__ __forceinline__ int64_t elem_signed(const uint8_t* p, int ew, int64_t i) {
  return ew == 8 ? reinterpret_cast<const int64_t*>(p)[i] : ew == 4 ? (int64_t)reinterpret_cast<const int32_t*>(p)[i]
                                                                     : (int64_t)reinterpret_cast<const int16_t*>(p)[i];
}
__device__ __forceinline__ uint64_t trunc_bits(uint64_t v, int ew) { return ew == 8 ? v : v & ((1ull << (8 * ew)) - 1); }

// pass 1: distinct bit patterns (dictionary jobs) or [lo, hi] (frame of reference) of one column of one batch
__global__ void __launch_bounds__(IMG_THREADS) image_analyse_kernel(ImageJob* jobs, uint64_t* tables) {
  ImageJob& j = jobs[blockIdx.x];
  __shared__ uint64_t set[SET_SLOTS];
  __shared__ uint64_t list[IMG_DICT_MAX + 1];
  __shared__ int cnt, over, has_empty, nlist;
  __shared__ long long rlo[IMG_THREADS / 32], rhi[IMG_THREADS / 32];
  const int tid = threadIdx.x;
  if (!j.dict) {
    long long lo = LLONG_MAX, hi = LLONG_MIN;
    for (int64_t i = tid; i < j.n; i += IMG_THREADS) { const long long v = elem_signed(j.src, j.ew, i); lo = min(lo, v); hi = max(hi, v); }
    for (int d = 16; d; d >>= 1) { lo = min(lo, __shfl_xor_sync(~0u, lo, d)); hi = max(hi, __shfl_xor_sync(~0u, hi, d)); }
    if ((tid & 31) == 0) { rlo[tid >> 5] = lo; rhi[tid >> 5] = hi; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < IMG_THREADS / 32; w++) { lo = min(lo, rlo[w]); hi = max(hi, rhi[w]); }
      j.lo = lo; j.hi = hi;
      j.ndict = 1;
    }
    return;
  }
  for (int i = tid; i < SET_SLOTS; i += IMG_THREADS) set[i] = SET_EMPTY;
  if (tid == 0) { cnt = 0; over = 0; has_empty = 0; nlist = 0; }
  __syncthreads();
  uint64_t last = 0;   // consecutive equal values cost no probe
  bool have_last = false;
  for (int64_t i = tid; i < j.n; i += IMG_THREADS) {
    if (*(volatile int*)&over) break;
    const uint64_t v = elem_bits(j.src, j.ew, i);
    if (have_last && v == last) continue;
    last = v;
    have_last = true;
    if (v == SET_EMPTY) { has_empty = 1; continue; }   // the sentinel itself (a NaN payload or -1) is counted apart
    uint32_t h = (uint32_t)((v * 0x9E3779B97F4A7C15ull) >> 55) & (SET_SLOTS - 1);
    for (int probe = 0;; probe++, h = (h + 1) & (SET_SLOTS - 1)) {
      if (probe == SET_SLOTS) { over = 1; break; }
      uint64_t cur = set[h];
      if (cur == v) break;
      if (cur == SET_EMPTY) {
        cur = atomicCAS(reinterpret_cast<unsigned long long*>(&set[h]), SET_EMPTY, v);
        if (cur == SET_EMPTY) { if (atomicAdd(&cnt, 1) >= IMG_DICT_MAX) over = 1; break; }
        if (cur == v) break;
      }
    }
  }
  __syncthreads();
  const int n = cnt + has_empty;
  if (over || n > IMG_DICT_MAX) {
    if (tid == 0) j.ndict = IMG_DICT_MAX + 1;
    return;
  }
  for (int i = tid; i < SET_SLOTS; i += IMG_THREADS) if (set[i] != SET_EMPTY) list[atomicAdd(&nlist, 1)] = set[i];
  if (tid == 0 && has_empty) list[atomicAdd(&nlist, 1)] = SET_EMPTY;
  __syncthreads();
  // sorted by bit pattern: the table (and so every code) does not depend on the order the set was filled in
  for (int i = tid; i < n; i += IMG_THREADS) {
    int rank = 0;
    for (int k = 0; k < n; k++) rank += list[k] < list[i];
    tables[(size_t)blockIdx.x * IMG_DICT_MAX + rank] = list[i];
  }
  if (tid == 0) j.ndict = n;
}

// pass 2: write the image and its table, then decode every row back from them and compare with the verbatim bytes
__global__ void __launch_bounds__(IMG_THREADS) image_encode_kernel(ImageJob* jobs, const uint64_t* tables) {
  ImageJob& j = jobs[blockIdx.x];
  if (!j.img) return;
  __shared__ uint64_t tab[IMG_DICT_MAX];
  __shared__ unsigned long long bad;
  const int tid = threadIdx.x;
  const int nd = j.dict ? j.ndict : 1, w = j.width;
  for (int i = tid; i < nd; i += IMG_THREADS) {
    tab[i] = j.dict ? tables[(size_t)blockIdx.x * IMG_DICT_MAX + i] : (uint64_t)j.lo;
    j.tab[i] = tab[i];
  }
  if (tid == 0) bad = 0;
  __syncthreads();
  for (int64_t i = tid; i < j.n; i += IMG_THREADS) {
    uint32_t code;
    if (j.dict) {   // binary search of the sorted table
      const uint64_t v = elem_bits(j.src, j.ew, i);
      int a = 0, b = nd - 1;
      while (a < b) { const int m = (a + b) >> 1; if (tab[m] < v) a = m + 1; else b = m; }
      code = (uint32_t)a;
    } else {
      code = (uint32_t)((uint64_t)elem_signed(j.src, j.ew, i) - (uint64_t)j.lo);
    }
    if (w == 1) j.img[i] = (uint8_t)code;
    else reinterpret_cast<uint16_t*>(j.img)[i] = (uint16_t)code;
  }
  __syncthreads();   // (the block's global writes are visible to the block past the barrier)
  unsigned long long mine = 0;
  const volatile uint64_t* vt = j.tab;
  for (int64_t i = tid; i < j.n; i += IMG_THREADS) {
    const volatile uint8_t* im = j.img;
    const uint32_t code = w == 1 ? im[i] : reinterpret_cast<const volatile uint16_t*>(im)[i];
    const uint64_t got = j.dict ? (code < (uint32_t)nd ? vt[code] : ~elem_bits(j.src, j.ew, i)) : trunc_bits(vt[0] + code, j.ew);
    if (got != elem_bits(j.src, j.ew, i)) mine++;
  }
  if (mine) atomicAdd(&bad, mine);
  __syncthreads();
  if (tid == 0) j.mismatches = (int64_t)bad;
}

// element bytes and image kind of a column the builder takes (0: none)
int image_source(const sd_column& sc, const StoredCol& c, bool* dict) {
  if (!c.present || !c.unsupported.empty() || c.has_nulls || c.dev.nulls || c.dev.img || !c.dev.data) return 0;
  *dict = false;
  switch (sc.type) {
    case SD_DOUBLE: *dict = true; return c.dev.enc == ENC_UNCOMPRESSED ? 8 : 0;
    case SD_FLOAT: *dict = true; return c.dev.enc == ENC_UNCOMPRESSED ? 4 : 0;
    case SD_LONG: case SD_TIMESTAMP: return c.dev.enc == ENC_UNCOMPRESSED ? 8 : 0;
    case SD_INT: case SD_DATE: return c.dev.enc == ENC_UNCOMPRESSED ? 4 : 0;
    case SD_SHORT: return c.dev.enc == ENC_UNCOMPRESSED ? 2 : 0;
    case SD_STRING: return c.dev.enc == ENC_DICTIONARY ? 2 : c.dev.enc == ENC_BIG_DICTIONARY ? 4 : 0;
    default: return 0;
  }
}

}  // namespace

int build_images(sd_store* s, cudaStream_t st, const std::vector<StoredBatch*>& batches, bool locked) {
  const auto t0 = std::chrono::steady_clock::now();
  if (const char* e = getenv("SD_TUNE_NO_SCAN_IMAGES")) if (atoi(e) > 0) return 0;   // (measurement aid: ingest without the build)
  std::vector<ImageJob> jobs;
  std::vector<std::pair<StoredBatch*, int>> where;
  for (StoredBatch* b : batches) {
    for (int c = 0; c < (int)b->cols.size() && c < (int)s->schema.size(); c++) {
      bool dict = false;
      const int ew = b->positional ? 0 : image_source(s->schema[c], b->cols[c], &dict);
      if (!ew || b->num_rows < IMG_MIN_ROWS) continue;
      ImageJob j;
      memset(&j, 0, sizeof(j));
      j.src = b->cols[c].dev.data; j.n = b->num_rows; j.ew = ew; j.dict = dict ? 1 : 0;
      jobs.push_back(j);
      where.emplace_back(b, c);
    }
  }
  if (jobs.empty()) return 0;
  const size_t nj = jobs.size();
  ImageJob* d_jobs = nullptr;
  uint64_t* d_tables = nullptr;
  SD_CUDA(cudaMallocAsync(&d_jobs, nj * sizeof(ImageJob), st));
  SD_CUDA(cudaMallocAsync(&d_tables, nj * IMG_DICT_MAX * 8, st));
  struct Free { cudaStream_t st; void* a; void* b; ~Free() { cudaFreeAsync(a, st); cudaFreeAsync(b, st); } } fr{st, d_jobs, d_tables};
  SD_CUDA(cudaMemcpyAsync(d_jobs, jobs.data(), nj * sizeof(ImageJob), cudaMemcpyHostToDevice, st));
  image_analyse_kernel<<<(unsigned)nj, IMG_THREADS, 0, st>>>(d_jobs, d_tables);
  SD_CUDA(cudaGetLastError());
  SD_CUDA(cudaMemcpyAsync(jobs.data(), d_jobs, nj * sizeof(ImageJob), cudaMemcpyDeviceToHost, st));
  SD_CUDA(cudaStreamSynchronize(st));
  // placement: [table, 128-byte aligned][codes + 128 bytes of slack for the bulk copies' 16-byte over-read]
  bool any = false;
  std::unique_lock<std::mutex> lock(s->mu, std::defer_lock);
  if (!locked) lock.lock();
  for (size_t i = 0; i < nj; i++) {
    ImageJob& j = jobs[i];
    j.width = image_width(j.dict != 0, j.ew, (uint64_t)j.ndict, j.lo, j.hi);
    if (!j.width) continue;
    const size_t tab_bytes = ((size_t)(j.dict ? j.ndict : 1) * 8 + 127) & ~size_t(127);
    const size_t bytes = tab_bytes + (size_t)j.n * j.width + 128;
    std::vector<Extent>* const outer = s->arena.record;   // (a caller's recorder stays in force afterwards)
    s->arena.record = &where[i].first->extents;
    uint8_t* p = s->arena.alloc(bytes, 128);
    s->arena.record = outer;
    if (!p) return SD_ERR_CUDA;
    j.tab = reinterpret_cast<uint64_t*>(p);
    j.img = p + tab_bytes;
    where[i].first->cols[where[i].second].img_bytes = (int64_t)bytes;
    any = true;
  }
  if (!locked) lock.unlock();
  if (!any) return 0;
  SD_CUDA(cudaMemcpyAsync(d_jobs, jobs.data(), nj * sizeof(ImageJob), cudaMemcpyHostToDevice, st));
  image_encode_kernel<<<(unsigned)nj, IMG_THREADS, 0, st>>>(d_jobs, d_tables);
  SD_CUDA(cudaGetLastError());
  std::vector<ImageJob> done(nj);
  SD_CUDA(cudaMemcpyAsync(done.data(), d_jobs, nj * sizeof(ImageJob), cudaMemcpyDeviceToHost, st));
  SD_CUDA(cudaStreamSynchronize(st));
  for (size_t i = 0; i < nj; i++) {
    const ImageJob& j = done[i];
    if (!j.img) continue;
    StoredCol& c = where[i].first->cols[where[i].second];
    if (j.mismatches) { if (!locked) lock.lock(); s->image_mismatches++; if (!locked) lock.unlock(); c.img_bytes = 0; continue; }   // the column keeps its verbatim path
    c.dev.img = j.img;
    c.dev.img_tab = j.tab;
    c.dev.img_w = j.width;
    c.dev.img_n = j.dict ? j.ndict : 1;
    c.img_ew = j.ew;
    c.img_dict = j.dict != 0;
  }
  if (!locked) lock.lock();
  s->image_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  return 0;
}

}  // namespace sd

extern "C" {

int sdx_store_image_info(sd_store* s, int64_t out[4]) {
  if (!s || !out) return sd::set_error(SD_ERR_INVALID, "sdx_store_image_info: null argument");
  std::lock_guard<std::mutex> lock(s->mu);
  out[0] = out[1] = 0;
  for (const auto& b : s->batches)
    for (const sd::StoredCol& c : b->cols)
      if (c.present && c.dev.img) { out[0] += c.img_bytes; out[1]++; }
  out[2] = s->image_mismatches;
  out[3] = (int64_t)(s->image_ms * 1000.0);
  return 0;
}

int sdx_image_width(int32_t dict, int32_t elem_bytes, uint64_t ndistinct, int64_t lo, int64_t hi, int32_t* width) {
  if (!width || (elem_bytes != 2 && elem_bytes != 4 && elem_bytes != 8)) return sd::set_error(SD_ERR_INVALID, "sdx_image_width: bad arguments");
  *width = sd::image_width(dict != 0, elem_bytes, ndistinct, lo, hi);
  return 0;
}

}  // extern "C"
