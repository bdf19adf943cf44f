// hbm_ceiling.cu -- how fast this GPU can read the bytes of the Q1 scan, without the scan's work.
//
// Every variant reads the same number of bytes as one SF-100 Q1 launch (600,037,902 rows x 40 B) and reduces them to one
// word so the loads cannot be dropped.  Kernel time from CUDA events, one variant per process (tools/hbm_ceiling.py runs
// them and samples the SM clock beside each):
//   r1      one contiguous buffer, grid-stride ld.global.cs.v4 (what the card can deliver at all)
//   r2      the same bytes as Q1's seven column streams (4 x 8 B, 2 x 2 B, 4 B per row) in 200,000-row batches placed like
//           sd_store places them (value start 128-byte aligned, 160 bytes of tail padding, 512 MB slabs); 8192-row chunks
//           dealt round-robin over a persistent grid, each 1024-row tile of every column read with direct v4 loads
//           (what the access pattern costs)
//   r3      r2's bytes through the scan kernel's producer pattern: one cp.async.bulk per column per 1024-row tile into an
//           mbarrier ring (same stage layout, same chunk order, 256 consumer threads + 1 producer warp, 1 CTA per SM);
//           consumers only release stages (what is left for the consumers' work)
//   r3lds   r3, and the consumers also read their rows of every column out of the stage (the scan's LDS, no arithmetic)
//
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o hbm_ceiling hbm_ceiling.cu
// usage: hbm_ceiling <r1|r2|r3|r3lds> [--ctas-per-sm N] [--stages N] [--reps N] [--warmup N]
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); exit(1); } } while (0)

constexpr int64_t ROWS = 600037902;      // TPC-H SF-100 lineitem
constexpr int ROWS_PER_BATCH = 200000;   // bench.py's batch size
constexpr int NC = 7;                     // Q1's scan columns, table order: quantity, extendedprice, discount, tax, returnflag, linestatus, shipdate
__host__ __device__ constexpr int width(int c) { return c < 4 ? 8 : c < 6 ? 2 : 4; }
__host__ __device__ constexpr int stage_width(int c) { return c < 4 ? 8 : 4; }   // the scan's stage slot per row (a dictionary-code slot holds int32)
constexpr int HEADER[NC] = {8, 8, 8, 8, 24, 20, 8};      // typeId + nulls size (+ dictionary of a code column) before the values
constexpr int THREADS = 256, RPT = 4, TILE_ROWS = THREADS * RPT, CHUNK_ROWS = 8192, MAX_STAGES = 12;
constexpr size_t SLAB = size_t(512) << 20;

struct Batch { const uint8_t* data[NC]; int32_t rows; int32_t pad; };

__device__ __forceinline__ uint32_t fold(uint4 v) { return v.x ^ v.y ^ v.z ^ v.w; }
__device__ __forceinline__ void publish(uint32_t x, unsigned* out) {
  for (int d = 16; d > 0; d >>= 1) x ^= __shfl_xor_sync(0xffffffffu, x, d);
  if ((threadIdx.x & 31) == 0) atomicXor(out, x);
}

// ---- r1 -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(512) r1_kernel(const uint4* p, int64_t n16, unsigned* out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t x = 0;
  for (; i + 3 * stride < n16; i += 4 * stride) {
    const uint4 a = __ldcs(p + i), b = __ldcs(p + i + stride), c = __ldcs(p + i + 2 * stride), d = __ldcs(p + i + 3 * stride);
    x ^= fold(a) ^ fold(b) ^ fold(c) ^ fold(d);
  }
  for (; i < n16; i += stride) x ^= fold(__ldcs(p + i));
  publish(x, out);
}

// ---- r2 -------------------------------------------------------------------------------------------
__device__ __forceinline__ int find_batch(const int32_t* prefix, int nb, int item) {
  int lo = 0, hi = nb;
  while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (prefix[mid] <= item) lo = mid; else hi = mid; }
  return lo;
}
__global__ void __launch_bounds__(THREADS) r2_kernel(const Batch* batches, const int32_t* prefix, int nb, int items, unsigned* out) {
  uint32_t x = 0;
  for (int item = blockIdx.x; item < items; item += gridDim.x) {
    const int bi = find_batch(prefix, nb, item);
    const Batch& b = batches[bi];
    const int rows = b.rows;
    const int t0 = (item - prefix[bi]) * CHUNK_ROWS;
    const int t1 = min(t0 + CHUNK_ROWS, rows);
    const uint8_t* base[NC];
#pragma unroll
    for (int c = 0; c < NC; c++) base[c] = b.data[c];
    for (int ts = t0; ts < t1; ts += TILE_ROWS) {
      const int r = min(TILE_ROWS, rows - ts);
      uint4 v[NC][2];
#pragma unroll
      for (int c = 0; c < NC; c++) {
        const int n16 = (r * width(c) + 15) / 16;
        const uint4* p = reinterpret_cast<const uint4*>(base[c] + (int64_t)ts * width(c));
#pragma unroll
        for (int k = 0; k < 2; k++) {
          const int j = threadIdx.x + k * THREADS;
          v[c][k] = j < n16 ? __ldcs(p + j) : make_uint4(0, 0, 0, 0);
        }
      }
#pragma unroll
      for (int c = 0; c < NC; c++) x ^= fold(v[c][0]) ^ fold(v[c][1]);
    }
  }
  publish(x, out);
}

// ---- r3 / r3lds: the scan's ring ----------------------------------------------------------------------
__host__ __device__ constexpr int stage_col_off(int c) {
  int off = 0;
  for (int i = 0; i < c; i++) off += TILE_ROWS * stage_width(i) + 128;
  return off;
}
constexpr int STAGE_BYTES = stage_col_off(NC);

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

template <bool LDS>
__global__ void __launch_bounds__(THREADS + 32, 1) r3_kernel(const Batch* batches, const int32_t* prefix, int nb, int items, int nstages,
                                                            unsigned* out) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem);
  uint64_t* empty_bar = full_bar + MAX_STAGES;
  uint8_t* ring = smem + 2 * MAX_STAGES * 8 + 64;   // stage regions 128-byte aligned (dynamic smem starts 1024-aligned)
  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int i = 0; i < nstages; i++) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], THREADS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid >= THREADS) {
    if (tid == THREADS) {
      int stage = 0;
      uint32_t phase = 0;
      for (int item = blockIdx.x; item < items; item += gridDim.x) {
        const int bi = find_batch(prefix, nb, item);
        const Batch& b = batches[bi];
        const int rows = b.rows;
        const int t0 = (item - prefix[bi]) * CHUNK_ROWS, t1 = min(t0 + CHUNK_ROWS, rows);
        const uint8_t* base[NC];
#pragma unroll
        for (int c = 0; c < NC; c++) base[c] = b.data[c];
        for (int ts = t0; ts < t1; ts += TILE_ROWS) {
          const int r = min(TILE_ROWS, rows - ts);
          uint32_t bytes[NC], total = 0;
#pragma unroll
          for (int c = 0; c < NC; c++) { bytes[c] = (uint32_t)((r * width(c) + 15) & ~15); total += bytes[c]; }
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          uint8_t* st = ring + (size_t)stage * STAGE_BYTES;
          mbar_expect_tx(&full_bar[stage], total);
#pragma unroll
          for (int c = 0; c < NC; c++) bulk_g2s(st + stage_col_off(c), base[c] + (int64_t)ts * width(c), bytes[c], &full_bar[stage]);
          if (++stage == nstages) { stage = 0; phase ^= 1u; }
        }
      }
    }
    return;
  }
  int stage = 0;
  uint32_t phase = 0;
  uint32_t x = 0;
  for (int item = blockIdx.x; item < items; item += gridDim.x) {
    const int bi = find_batch(prefix, nb, item);
    const int rows = batches[bi].rows;
    const int t0 = (item - prefix[bi]) * CHUNK_ROWS, t1 = min(t0 + CHUNK_ROWS, rows);
    for (int ts = t0; ts < t1; ts += TILE_ROWS) {
      mbar_wait(&full_bar[stage], phase);
      if (LDS) {   // the scan's consumer loads: row pair u of thread t at u * 2 * THREADS + 2 * t
        const uint8_t* st = ring + (size_t)stage * STAGE_BYTES;
#pragma unroll
        for (int u = 0; u < RPT / 2; u++) {
          const int p = u * 2 * THREADS + 2 * tid;
#pragma unroll
          for (int c = 0; c < NC; c++) {
            const uint8_t* q = st + stage_col_off(c) + p * width(c);
            if (width(c) == 8) { const uint4 v = *reinterpret_cast<const uint4*>(q); x ^= fold(v); }
            else if (width(c) == 4) { const uint2 v = *reinterpret_cast<const uint2*>(q); x ^= v.x ^ v.y; }
            else x ^= *reinterpret_cast<const uint32_t*>(q);
          }
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();
      if ((tid & 31) == 0) mbar_arrive(&empty_bar[stage]);
      if (++stage == nstages) { stage = 0; phase ^= 1u; }
    }
  }
  publish(x, out);
}

// ---- host ----------------------------------------------------------------------------------------------
int main(int argc, char** argv) {
  if (argc < 2) { fprintf(stderr, "usage: %s <r1|r2|r3|r3lds> [--ctas-per-sm N] [--stages N] [--reps N] [--warmup N]\n", argv[0]); return 2; }
  const std::string variant = argv[1];
  int ctas_per_sm = variant == "r1" ? 4 : variant == "r2" ? 4 : 1, nstages = 3, reps = 30, warmup = 60;
  for (int i = 2; i + 1 < argc; i += 2) {
    const std::string k = argv[i];
    const int v = atoi(argv[i + 1]);
    if (k == "--ctas-per-sm") ctas_per_sm = v;
    else if (k == "--stages") nstages = v;
    else if (k == "--reps") reps = v;
    else if (k == "--warmup") warmup = v;
    else { fprintf(stderr, "unknown option %s\n", k.c_str()); return 2; }
  }
  if (variant != "r1" && variant != "r2" && variant != "r3" && variant != "r3lds") { fprintf(stderr, "unknown variant %s\n", variant.c_str()); return 2; }
  if (nstages < 2 || nstages > MAX_STAGES || reps < 1) { fprintf(stderr, "bad --stages / --reps\n"); return 2; }

  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  const int sms = prop.multiProcessorCount;

  // placement: every column buffer of a batch bump-allocated in 512 MB slabs, value start 128-byte aligned, 160 bytes of
  // tail padding; r1 reads the first `algo` bytes of the same allocation contiguously
  const int nb = (int)((ROWS + ROWS_PER_BATCH - 1) / ROWS_PER_BATCH);
  std::vector<Batch> hb(nb);
  std::vector<int32_t> prefix(nb + 1, 0);
  size_t slab_base = 0, off = 0;
  int64_t algo = 0;
  std::vector<size_t> offs((size_t)nb * NC);
  for (int b = 0; b < nb; b++) {
    const int rows = (int)std::min<int64_t>(ROWS_PER_BATCH, ROWS - (int64_t)b * ROWS_PER_BATCH);
    hb[b].rows = rows;
    prefix[b + 1] = prefix[b] + (rows + CHUNK_ROWS - 1) / CHUNK_ROWS;
    for (int c = 0; c < NC; c++) {
      const size_t len = (size_t)HEADER[c] + (size_t)rows * width(c);
      size_t want = (slab_base + off + HEADER[c] + 127) / 128 * 128 - HEADER[c];
      if (want + len + 160 > slab_base + SLAB) { slab_base += SLAB; off = 0; want = (slab_base + HEADER[c] + 127) / 128 * 128 - HEADER[c]; }
      offs[(size_t)b * NC + c] = want + HEADER[c];
      off = want + len + 160 - slab_base;
      algo += (int64_t)rows * width(c);
    }
  }
  const size_t span = slab_base + off + 4096;
  uint8_t* d = nullptr;
  CK(cudaMalloc(&d, span));
  CK(cudaMemset(d, 0x5a, span));
  for (int b = 0; b < nb; b++)
    for (int c = 0; c < NC; c++) hb[b].data[c] = d + offs[(size_t)b * NC + c];
  Batch* d_batches = nullptr;
  int32_t* d_prefix = nullptr;
  unsigned* d_out = nullptr;
  CK(cudaMalloc(&d_batches, sizeof(Batch) * nb));
  CK(cudaMalloc(&d_prefix, sizeof(int32_t) * (nb + 1)));
  CK(cudaMalloc(&d_out, sizeof(unsigned)));
  CK(cudaMemcpy(d_batches, hb.data(), sizeof(Batch) * nb, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_prefix, prefix.data(), sizeof(int32_t) * (nb + 1), cudaMemcpyHostToDevice));
  CK(cudaMemset(d_out, 0, sizeof(unsigned)));
  const int items = prefix[nb];

  size_t smem = 0;
  if (variant == "r3" || variant == "r3lds") {
    smem = 2 * MAX_STAGES * 8 + 64 + (size_t)nstages * STAGE_BYTES;
    if (smem > (size_t)prop.sharedMemPerBlockOptin) { fprintf(stderr, "%d stages need %zu B of shared memory (max %zu)\n", nstages, smem, (size_t)prop.sharedMemPerBlockOptin); return 2; }
    CK(cudaFuncSetAttribute(r3_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CK(cudaFuncSetAttribute(r3_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  }
  const int grid = sms * ctas_per_sm;
  auto launch = [&]() {
    if (variant == "r1") r1_kernel<<<grid, 512>>>(reinterpret_cast<const uint4*>(d), (algo + 15) / 16, d_out);
    else if (variant == "r2") r2_kernel<<<grid, THREADS>>>(d_batches, d_prefix, nb, items, d_out);
    else if (variant == "r3") r3_kernel<false><<<sms, THREADS + 32, smem>>>(d_batches, d_prefix, nb, items, nstages, d_out);
    else r3_kernel<true><<<sms, THREADS + 32, smem>>>(d_batches, d_prefix, nb, items, nstages, d_out);
  };
  for (int i = 0; i < warmup; i++) launch();
  CK(cudaGetLastError());
  CK(cudaDeviceSynchronize());
  std::vector<cudaEvent_t> ev(2 * reps);
  for (auto& e : ev) CK(cudaEventCreate(&e));
  for (int i = 0; i < reps; i++) {
    CK(cudaEventRecord(ev[2 * i]));
    launch();
    CK(cudaEventRecord(ev[2 * i + 1]));
  }
  CK(cudaGetLastError());
  CK(cudaDeviceSynchronize());
  std::vector<float> ms(reps);
  for (int i = 0; i < reps; i++) CK(cudaEventElapsedTime(&ms[i], ev[2 * i], ev[2 * i + 1]));
  std::sort(ms.begin(), ms.end());
  unsigned h_out = 0;
  CK(cudaMemcpy(&h_out, d_out, sizeof(unsigned), cudaMemcpyDeviceToHost));
  const double med = ms[reps / 2], best = ms[0];
  printf("{\"variant\": \"%s\", \"grid\": %d, \"threads\": %d, \"stages\": %d, \"stage_bytes\": %d, \"smem\": %zu, \"bytes\": %lld, "
         "\"reps\": %d, \"ms_median\": %.4f, \"ms_min\": %.4f, \"ms_max\": %.4f, \"gbps_median\": %.1f, \"gbps_best\": %.1f, \"check\": %u}\n",
         variant.c_str(), variant.rfind("r3", 0) == 0 ? sms : grid, variant == "r1" ? 512 : variant == "r2" ? THREADS : THREADS + 32,
         variant.rfind("r3", 0) == 0 ? nstages : 0, STAGE_BYTES, smem, (long long)algo, reps, med, best, ms[reps - 1],
         algo / (med * 1e-3) / 1e9, algo / (best * 1e-3) / 1e9, h_out);
  for (auto& e : ev) cudaEventDestroy(e);
  cudaFree(d);
  cudaFree(d_batches);
  cudaFree(d_prefix);
  cudaFree(d_out);
  return 0;
}
