// sd_hash.cu -- housekeeping kernels of the MODE_HASH group table (init with slot identities, compaction
// of the occupied entries before the read-back).  The find-or-insert itself is in sd_kernels.cuh.
#include <algorithm>

#include "sd_host.h"

namespace sd {

__global__ void hash_init_kernel(uint32_t* state, uint64_t* vals, uint32_t capacity, int nslot, const uint64_t* ident) {
  const size_t n = (size_t)capacity * nslot;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) vals[i] = ident[i % nslot];
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < capacity; i += (size_t)gridDim.x * blockDim.x) state[i] = 0u;
}

__global__ void hash_compact_kernel(const uint32_t* state, const int64_t* keys, const uint32_t* knull, const uint64_t* vals,
                                    uint32_t capacity, int nk, int nslot, int64_t* out_keys, uint32_t* out_knull, uint64_t* out_vals,
                                    uint32_t* cursor, const uint64_t* shifts, int nshift, uint64_t* out_shifts) {
  for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < capacity; e += gridDim.x * blockDim.x) {
    if (state[e] != 2u) continue;
    const uint32_t o = atomicAdd(cursor, 1u);
    for (int k = 0; k < nk; k++) out_keys[(size_t)o * nk + k] = keys[(size_t)e * nk + k];
    out_knull[o] = knull[e];
    for (int s = 0; s < nslot; s++) out_vals[(size_t)o * nslot + s] = vals[(size_t)e * nslot + s];
    for (int s = 0; s < nshift; s++) out_shifts[(size_t)o * nshift + s] = shifts[(size_t)e * nshift + s];
  }
}

int hash_table_init(cudaStream_t stream, const HashTable& t, uint32_t capacity, int nslot, const uint64_t* d_ident, int nshift) {
  hash_init_kernel<<<296, 256, 0, stream>>>(t.state, t.vals, capacity, nslot, d_ident);
  SD_CUDA(cudaGetLastError());
  if (nshift > 0) SD_CUDA(cudaMemsetAsync(t.shifts, 0xff, (size_t)capacity * nshift * 8, stream));   // SHIFT_EMPTY
  SD_CUDA(cudaMemsetAsync(t.overflow, 0, 4, stream));
  SD_CUDA(cudaMemsetAsync(t.count, 0, 4, stream));
  return 0;
}

int hash_table_compact(cudaStream_t stream, const HashTable& t, uint32_t capacity, int nk, int nslot, int64_t* out_keys,
                       uint32_t* out_knull, uint64_t* out_vals, uint32_t* d_cursor, int nshift, uint64_t* out_shifts) {
  SD_CUDA(cudaMemsetAsync(d_cursor, 0, 4, stream));
  hash_compact_kernel<<<296, 256, 0, stream>>>(t.state, t.keys, t.knull, t.vals, capacity, nk, nslot, out_keys, out_knull, out_vals, d_cursor,
                                               t.shifts, nshift, out_shifts);
  SD_CUDA(cudaGetLastError());
  return 0;
}

// ---- strings held by reference (hash-table keys, projected raw strings) -> host -------------------------------------
__global__ void rec_lens_kernel(const int64_t* recs, int64_t n, int64_t stride, int32_t* lens) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint8_t* r = reinterpret_cast<const uint8_t*>(recs[i * stride]);
    lens[i] = r ? (int32_t)((uint32_t)r[0] | ((uint32_t)r[1] << 8) | ((uint32_t)r[2] << 16) | ((uint32_t)r[3] << 24)) : -1;
  }
}
__global__ void rec_bytes_kernel(const int64_t* recs, int64_t n, int64_t stride, const int64_t* offs, uint8_t* out) {
  // one warp per record
  const int lane = threadIdx.x & 31;
  for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const uint8_t* r = reinterpret_cast<const uint8_t*>(recs[i * stride]);
    if (!r) continue;
    const int64_t len = offs[i + 1] - offs[i];
    for (int64_t b = lane; b < len; b += 32) out[offs[i] + b] = r[4 + b];
  }
}

int fetch_string_records(cudaStream_t stream, const int64_t* d_recs, int64_t n, int64_t stride, std::vector<std::string>& out) {
  out.assign((size_t)n, std::string());
  if (n <= 0) return 0;
  int32_t* d_lens = nullptr;
  int64_t* d_offs = nullptr;
  uint8_t* d_bytes = nullptr;
  auto cleanup = [&]() { if (d_lens) cudaFree(d_lens); if (d_offs) cudaFree(d_offs); if (d_bytes) cudaFree(d_bytes); };
#define FSR(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { cleanup(); return set_error(SD_ERR_CUDA, "%s: %s", #call, cudaGetErrorString(e_)); } } while (0)
  FSR(cudaMalloc(&d_lens, (size_t)n * 4));
  const int blocks = (int)std::min<int64_t>(1184, (n + 255) / 256);
  rec_lens_kernel<<<blocks, 256, 0, stream>>>(d_recs, n, stride, d_lens);
  FSR(cudaGetLastError());
  std::vector<int32_t> lens((size_t)n);
  FSR(cudaMemcpyAsync(lens.data(), d_lens, (size_t)n * 4, cudaMemcpyDeviceToHost, stream));
  FSR(cudaStreamSynchronize(stream));
  std::vector<int64_t> offs((size_t)n + 1, 0);
  for (int64_t i = 0; i < n; i++) offs[(size_t)i + 1] = offs[(size_t)i] + (lens[(size_t)i] > 0 ? lens[(size_t)i] : 0);
  const int64_t total = offs[(size_t)n];
  if (total > 0) {
    FSR(cudaMalloc(&d_offs, ((size_t)n + 1) * 8));
    FSR(cudaMalloc(&d_bytes, (size_t)total));
    FSR(cudaMemcpyAsync(d_offs, offs.data(), ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, stream));
    rec_bytes_kernel<<<(int)std::min<int64_t>(1184, (n * 32 + 255) / 256), 256, 0, stream>>>(d_recs, n, stride, d_offs, d_bytes);
    FSR(cudaGetLastError());
    std::vector<uint8_t> bytes((size_t)total);
    FSR(cudaMemcpyAsync(bytes.data(), d_bytes, (size_t)total, cudaMemcpyDeviceToHost, stream));
    FSR(cudaStreamSynchronize(stream));
    for (int64_t i = 0; i < n; i++) if (lens[(size_t)i] > 0) out[(size_t)i].assign(reinterpret_cast<const char*>(bytes.data() + offs[(size_t)i]), (size_t)lens[(size_t)i]);
  }
#undef FSR
  cleanup();
  return 0;
}

}  // namespace sd
