// sd_gen.cu -- synthetic lineitem column batches generated on the device straight into a store
// (bench / test utility, `sdx_` prefix: not part of the reference boundary).
//
// Byte-identical to snappydata_b200/lineitem.py (tests/test_lineitem_gen.py checks it): every value is
// a pure function of (seed, global row, stream); string columns are Dictionary encoded with per-batch
// dictionaries in first-seen order, the rest Uncompressed, all NOT NULL -- what the reference's default
// encoders (enc/ColumnEncoding.scala:837-844) produce for TPCHTableSchema.scala:122-143.
#include <algorithm>
#include <climits>
#include <cstring>

#include "sd_host.h"

namespace {

using namespace sd;

__host__ __device__ inline uint64_t mix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__host__ __device__ inline uint64_t hrow(uint64_t row, int stream, uint64_t seed) { return mix64(seed ^ mix64(row * 16 + (uint64_t)stream)); }

__device__ inline int32_t gen_shipdate(uint64_t row, uint64_t seed) { return 8036 + (int32_t)(hrow(row, 4, seed) % 2526ull); }
// returnflag class: 0 'N', 1 'R', 2 'A'; linestatus class: 0 'O', 1 'F'
__device__ inline void gen_flags(uint64_t row, uint64_t seed, int32_t ship, int* rf, int* ls) {
  if (ship > 9298) { *rf = 0; *ls = 0; return; }
  const int r = (int)(hrow(row, 5, seed) % 100ull);
  *rf = r < 2 ? 0 : (r < 51 ? 1 : 2);
  *ls = 1;
}

struct GenBatch {
  uint64_t first_row;
  int32_t n;
  int32_t pad_;
  uint8_t* col[7];          // device buffer start of: qty, price, disc, tax, returnflag, linestatus, shipdate (or nullptr)
  int64_t body_off[7];
  uint8_t prefix[2][32];    // header + dictionary bytes of returnflag / linestatus
  int32_t prefix_len[2];
  int8_t rf_code[4];
  int8_t ls_code[4];
};

__global__ void first_seen_kernel(const uint64_t* first_rows, const int32_t* counts, uint64_t seed, int32_t* out) {
  __shared__ int first[5];
  const int b = blockIdx.x;
  if (threadIdx.x < 5) first[threadIdx.x] = INT_MAX;
  __syncthreads();
  const uint64_t r0 = first_rows[b];
  const int n = counts[b];
  int loc[5] = {INT_MAX, INT_MAX, INT_MAX, INT_MAX, INT_MAX};
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    int rf, ls;
    gen_flags(r0 + i, seed, gen_shipdate(r0 + i, seed), &rf, &ls);
    if (i < loc[rf]) loc[rf] = i;
    if (i < loc[3 + ls]) loc[3 + ls] = i;
  }
  for (int k = 0; k < 5; k++) if (loc[k] != INT_MAX) atomicMin(&first[k], loc[k]);
  __syncthreads();
  if (threadIdx.x < 5) out[b * 5 + threadIdx.x] = first[threadIdx.x];
}

constexpr int GEN_ROWS_PER_CTA = 4096;

__global__ void fill_kernel(const GenBatch* batches, const int32_t* chunk_prefix, int nbatches, uint64_t seed) {
  const int item = blockIdx.x;
  int lo = 0, hi = nbatches;
  while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (chunk_prefix[mid] <= item) lo = mid; else hi = mid; }
  const GenBatch& g = batches[lo];
  const int chunk = item - chunk_prefix[lo];
  if (chunk == 0) {   // headers / dictionaries
    if (threadIdx.x < 7 && g.col[threadIdx.x] && threadIdx.x != 4 && threadIdx.x != 5) {
      reinterpret_cast<int32_t*>(g.col[threadIdx.x])[0] = ENC_UNCOMPRESSED;   // typeId
      reinterpret_cast<int32_t*>(g.col[threadIdx.x])[1] = 0;                  // null bytes
    }
    for (int k = 0; k < 2; k++)
      if (g.col[4 + k] && (int)threadIdx.x < g.prefix_len[k]) g.col[4 + k][threadIdx.x] = g.prefix[k][threadIdx.x];
  }
  const int base = chunk * GEN_ROWS_PER_CTA;
  for (int p = base + 2 * (int)threadIdx.x; p < min(base + GEN_ROWS_PER_CTA, g.n); p += 2 * blockDim.x) {
    const int cnt = min(2, g.n - p);
    double q[2], pr[2], di[2], tx[2];
    int32_t sh[2];
    int16_t rfc[2], lsc[2];
    for (int j = 0; j < 2; j++) {
      const uint64_t row = g.first_row + (uint64_t)(p + (j < cnt ? j : 0));
      q[j] = (double)(1ull + hrow(row, 0, seed) % 50ull);
      pr[j] = (double)(90000ull + hrow(row, 1, seed) % 10410000ull) / 100.0;
      di[j] = (double)(hrow(row, 2, seed) % 11ull) / 100.0;
      tx[j] = (double)(hrow(row, 3, seed) % 9ull) / 100.0;
      sh[j] = gen_shipdate(row, seed);
      int rf, ls;
      gen_flags(row, seed, sh[j], &rf, &ls);
      rfc[j] = g.rf_code[rf];
      lsc[j] = g.ls_code[ls];
    }
    if (cnt == 2) {
      if (g.col[0]) *reinterpret_cast<double2*>(g.col[0] + g.body_off[0] + 8ll * p) = make_double2(q[0], q[1]);
      if (g.col[1]) *reinterpret_cast<double2*>(g.col[1] + g.body_off[1] + 8ll * p) = make_double2(pr[0], pr[1]);
      if (g.col[2]) *reinterpret_cast<double2*>(g.col[2] + g.body_off[2] + 8ll * p) = make_double2(di[0], di[1]);
      if (g.col[3]) *reinterpret_cast<double2*>(g.col[3] + g.body_off[3] + 8ll * p) = make_double2(tx[0], tx[1]);
      if (g.col[6]) *reinterpret_cast<int2*>(g.col[6] + g.body_off[6] + 4ll * p) = make_int2(sh[0], sh[1]);
      if (g.col[4]) *reinterpret_cast<uint32_t*>(g.col[4] + g.body_off[4] + 2ll * p) = (uint32_t)(uint16_t)rfc[0] | ((uint32_t)(uint16_t)rfc[1] << 16);
      if (g.col[5]) *reinterpret_cast<uint32_t*>(g.col[5] + g.body_off[5] + 2ll * p) = (uint32_t)(uint16_t)lsc[0] | ((uint32_t)(uint16_t)lsc[1] << 16);
    } else {
      if (g.col[0]) *reinterpret_cast<double*>(g.col[0] + g.body_off[0] + 8ll * p) = q[0];
      if (g.col[1]) *reinterpret_cast<double*>(g.col[1] + g.body_off[1] + 8ll * p) = pr[0];
      if (g.col[2]) *reinterpret_cast<double*>(g.col[2] + g.body_off[2] + 8ll * p) = di[0];
      if (g.col[3]) *reinterpret_cast<double*>(g.col[3] + g.body_off[3] + 8ll * p) = tx[0];
      if (g.col[6]) *reinterpret_cast<int32_t*>(g.col[6] + g.body_off[6] + 4ll * p) = sh[0];
      if (g.col[4]) *reinterpret_cast<int16_t*>(g.col[4] + g.body_off[4] + 2ll * p) = rfc[0];
      if (g.col[5]) *reinterpret_cast<int16_t*>(g.col[5] + g.body_off[5] + 2ll * p) = lsc[0];
    }
  }
}

// table ordinals of the 7 generated columns, in GenBatch.col order
const int kOrdinal[7] = {4, 5, 6, 7, 8, 9, 10};
const int kType[7] = {SD_DOUBLE, SD_DOUBLE, SD_DOUBLE, SD_DOUBLE, SD_STRING, SD_STRING, SD_DATE};

}  // namespace

extern "C" int sdx_store_gen_lineitem(sd_store* s, int64_t first_row, int64_t nrows, int32_t rows_per_batch, int32_t nbuckets,
                                      uint64_t seed, int32_t column_mask) {
  using namespace sd;
  if (!s || nrows < 0 || rows_per_batch <= 0 || nbuckets <= 0) return set_error(SD_ERR_INVALID, "sdx_store_gen_lineitem: bad arguments");
  if (first_row % rows_per_batch) return set_error(SD_ERR_INVALID, "first_row must be a multiple of rows_per_batch");
  if (s->schema.size() < 11) return set_error(SD_ERR_INVALID, "store schema is not lineitem (needs >= 11 columns)");
  for (int k = 0; k < 7; k++)
    if ((column_mask >> kOrdinal[k]) & 1)
      if (s->schema[kOrdinal[k]].type != kType[k] || s->schema[kOrdinal[k]].nullable)
        return set_error(SD_ERR_INVALID, "store schema column %d does not match lineitem", kOrdinal[k]);
  if (nrows == 0) return 0;
  std::lock_guard<std::mutex> lock(s->mu);
  SD_CUDA(cudaSetDevice(s->device));
  const int nb = (int)((nrows + rows_per_batch - 1) / rows_per_batch);
  std::vector<uint64_t> firsts(nb);
  std::vector<int32_t> counts(nb), prefix(nb + 1, 0);
  for (int b = 0; b < nb; b++) {
    firsts[b] = (uint64_t)first_row + (uint64_t)b * rows_per_batch;
    counts[b] = (int32_t)std::min<int64_t>(rows_per_batch, nrows - (int64_t)b * rows_per_batch);
    prefix[b + 1] = prefix[b] + (counts[b] + GEN_ROWS_PER_CTA - 1) / GEN_ROWS_PER_CTA;
  }
  uint64_t* d_firsts; int32_t *d_counts, *d_first_seen, *d_prefix; GenBatch* d_gen;
  SD_CUDA(cudaMalloc(&d_firsts, nb * 8));
  SD_CUDA(cudaMalloc(&d_counts, nb * 4));
  SD_CUDA(cudaMalloc(&d_first_seen, nb * 20));
  SD_CUDA(cudaMalloc(&d_prefix, (nb + 1) * 4));
  SD_CUDA(cudaMalloc(&d_gen, sizeof(GenBatch) * (size_t)nb));
  SD_CUDA(cudaMemcpy(d_firsts, firsts.data(), nb * 8, cudaMemcpyHostToDevice));
  SD_CUDA(cudaMemcpy(d_counts, counts.data(), nb * 4, cudaMemcpyHostToDevice));
  SD_CUDA(cudaMemcpy(d_prefix, prefix.data(), (nb + 1) * 4, cudaMemcpyHostToDevice));
  first_seen_kernel<<<nb, 256, 0, s->copy_stream>>>(d_firsts, d_counts, seed, d_first_seen);
  std::vector<int32_t> fs((size_t)nb * 5);
  SD_CUDA(cudaMemcpyAsync(fs.data(), d_first_seen, (size_t)nb * 20, cudaMemcpyDeviceToHost, s->copy_stream));
  SD_CUDA(cudaStreamSynchronize(s->copy_stream));

  static const char* rf_str[3] = {"N", "R", "A"};
  static const char* ls_str[2] = {"O", "F"};
  std::vector<GenBatch> gen(nb);
  const size_t first_batch = s->batches.size();
  std::vector<StoredBatch*> fresh;
  for (int b = 0; b < nb; b++) {
    GenBatch& g = gen[b];
    memset(&g, 0, sizeof(g));
    g.first_row = firsts[b];
    g.n = counts[b];
    std::unique_ptr<StoredBatch> sb(new StoredBatch());
    sb->num_rows = counts[b];
    sb->batch_id = (int64_t)(firsts[b] / rows_per_batch);
    sb->bucket_id = (int32_t)(sb->batch_id % nbuckets);
    sb->cols.resize(s->schema.size());
    ExtentRecorder rec(s->arena, &sb->extents);
    for (int k = 0; k < 7; k++) {
      if (!((column_mask >> kOrdinal[k]) & 1)) continue;
      StoredCol& c = sb->cols[kOrdinal[k]];
      c.present = true;
      memset(&c.dev, 0, sizeof(c.dev));
      int64_t body, len;
      if (k == 4 || k == 5) {   // dictionary in first-seen order
        const int nvals = k == 4 ? 3 : 2;
        const int32_t* f = &fs[(size_t)b * 5 + (k == 4 ? 0 : 3)];
        int order[3] = {0, 1, 2};
        std::sort(order, order + nvals, [&](int x, int y) { return f[x] < f[y]; });
        int8_t* code = k == 4 ? g.rf_code : g.ls_code;
        uint8_t* pre = g.prefix[k - 4];
        int pl = 0, nd = 0;
        const int32_t enc = ENC_DICTIONARY, zero = 0;
        memcpy(pre, &enc, 4); memcpy(pre + 4, &zero, 4); pl = 12;   // [typeId][nullBytes][numElements]
        for (int j = 0; j < nvals; j++) {
          const int v = order[j];
          if (f[v] == INT_MAX) continue;
          code[v] = (int8_t)nd++;
          const char* str = k == 4 ? rf_str[v] : ls_str[v];
          const int32_t one = 1;
          c.dict_rec_off.push_back(pl);
          memcpy(pre + pl, &one, 4); pre[pl + 4] = (uint8_t)str[0]; pl += 5;
          c.dict_strings.push_back(std::string(str, 1));
        }
        memcpy(pre + 8, &nd, 4);
        g.prefix_len[k - 4] = pl;
        body = pl;
        len = body + 2ll * counts[b];
        c.dev.enc = ENC_DICTIONARY;
        c.dev.dict_n = nd;
        c.algo_bytes = len - 8 - (pl - 8);
      } else {
        body = 8;
        len = body + (k == 6 ? 4ll : 8ll) * counts[b];
        c.dev.enc = ENC_UNCOMPRESSED;
        c.algo_bytes = len - 8;
      }
      c.len = len;
      c.body_off = body;
      c.dev_base = s->arena.alloc((size_t)len + 160, 128, (size_t)body);
      if (!c.dev_base) return SD_ERR_CUDA;
      c.dev.data = c.dev_base + body;
      for (size_t e = 0; e < c.dict_rec_off.size(); e++) c.dict_rec_ptr.push_back((int64_t)(uintptr_t)(c.dev_base + c.dict_rec_off[e]));
      c.fast = true;
      g.col[k] = c.dev_base;
      g.body_off[k] = body;
    }
    fresh.push_back(sb.get());
    s->batches.push_back(std::move(sb));
  }
  (void)first_batch;
  SD_CUDA(cudaMemcpyAsync(d_gen, gen.data(), sizeof(GenBatch) * (size_t)nb, cudaMemcpyHostToDevice, s->copy_stream));
  fill_kernel<<<prefix[nb], 256, 0, s->copy_stream>>>(d_gen, d_prefix, nb, seed);
  SD_CUDA(cudaGetLastError());
  SD_CUDA(cudaStreamSynchronize(s->copy_stream));
  cudaFree(d_firsts); cudaFree(d_counts); cudaFree(d_first_seen); cudaFree(d_prefix); cudaFree(d_gen);
  { int rc = build_images(s, s->copy_stream, fresh, true); if (rc) return rc; }
  s->version++;
  return 0;
}
