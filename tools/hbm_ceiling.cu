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
// Two more dimensions say whether Hopper's generic memory compression (done by the hardware between L2 and DRAM, invisible
// to kernels) lowers the DRAM bytes behind those reads:
//   --alloc plain          one cudaMalloc (never compressible)
//   --alloc compressible   512 MB chunks from cuMemCreate with allocFlags.compressionType = CU_MEM_ALLOCATION_COMP_GENERIC,
//                          mapped back to back into one reserved range; what the driver granted is read back per chunk
//   --fill const           every byte 0x5a (the positive control: the most compressible content there is)
//   --fill random          splitmix64 bytes (the negative control)
//   --fill q1              every column stream holds the lineitem generator's values (snappydata_b200/lineitem.py; the
//                          dictionary codes are the flag classes, the same {0,1,2} value set the store's codes take)
//   --fill q1:<column>     only that column holds generator values, the others random bytes (which columns compress)
//
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o hbm_ceiling hbm_ceiling.cu
// usage: hbm_ceiling <r1|r2|r3|r3lds> [--ctas-per-sm N] [--stages N] [--reps N] [--warmup N] [--alloc plain|compressible]
//                    [--fill const|random|q1|q1:<column>]
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); exit(1); } } while (0)
#define CU(x) do { CUresult r_ = (x); if (r_ != CUDA_SUCCESS) { fprintf(stderr, "%s:%d %s: CUresult %d\n", __FILE__, __LINE__, #x, (int)r_); exit(1); } } while (0)

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

// ---- fills --------------------------------------------------------------------------------------------
__host__ __device__ inline uint64_t mix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__device__ inline uint64_t hrow(uint64_t row, int stream, uint64_t seed) { return mix64(seed ^ mix64(row * 16 + (uint64_t)stream)); }

__global__ void random_fill_kernel(uint64_t* p, int64_t n8) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (int64_t)gridDim.x * blockDim.x) p[i] = mix64(~(uint64_t)i);
}

// column c of every row: the generator's value where bit c of `mask` is set, random bytes elsewhere
__global__ void q1_fill_kernel(const Batch* batches, int mask, uint64_t seed) {
  for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < ROWS; row += (int64_t)gridDim.x * blockDim.x) {
    const Batch& b = batches[row / ROWS_PER_BATCH];
    const int64_t i = row % ROWS_PER_BATCH;
    const uint64_t r = (uint64_t)row;
    const int32_t ship = 8036 + (int32_t)(hrow(r, 4, seed) % 2526ull);
    const int fr = (int)(hrow(r, 5, seed) % 100ull);
    const int16_t rf = ship > 9298 ? 0 : fr < 2 ? 0 : fr < 51 ? 1 : 2, ls = ship > 9298 ? 0 : 1;
    const double q = (double)(1ull + hrow(r, 0, seed) % 50ull), pr = (double)(90000ull + hrow(r, 1, seed) % 10410000ull) / 100.0;
    const double di = (double)(hrow(r, 2, seed) % 11ull) / 100.0, tx = (double)(hrow(r, 3, seed) % 9ull) / 100.0;
    const double dv[4] = {q, pr, di, tx};
#pragma unroll
    for (int c = 0; c < NC; c++) {
      const uint64_t junk = mix64(~(r * NC + c));
      uint8_t* dst = const_cast<uint8_t*>(b.data[c]) + i * width(c);
      const bool gen = (mask >> c) & 1;
      if (width(c) == 8) *reinterpret_cast<uint64_t*>(dst) = gen ? (uint64_t)__double_as_longlong(dv[c < 4 ? c : 0]) : junk;
      else if (width(c) == 4) *reinterpret_cast<int32_t*>(dst) = gen ? ship : (int32_t)junk;
      else *reinterpret_cast<int16_t*>(dst) = gen ? (c == 4 ? rf : ls) : (int16_t)junk;
    }
  }
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
static const char* const COLUMN_NAMES[NC] = {"quantity", "extendedprice", "discount", "tax", "returnflag", "linestatus", "shipdate"};

// compressible memory: the driver entry points through the runtime, so the probe needs no -lcuda
struct Vmm {
  PFN_cuMemCreate_v10020 create;
  PFN_cuMemRelease_v10020 release;
  PFN_cuMemAddressReserve_v10020 reserve;
  PFN_cuMemAddressFree_v10020 free_range;
  PFN_cuMemMap_v10020 map;
  PFN_cuMemUnmap_v10020 unmap;
  PFN_cuMemSetAccess_v10020 set_access;
  PFN_cuMemGetAllocationGranularity_v10020 granularity;
  PFN_cuMemGetAllocationPropertiesFromHandle_v10020 props;
  PFN_cuDeviceGetAttribute_v2000 attribute;
  void load() {
    auto get = [](const char* name, void** fn) {
      cudaDriverEntryPointQueryResult q;
      CK(cudaGetDriverEntryPointByVersion(name, fn, 12000, cudaEnableDefault, &q));
      if (q != cudaDriverEntryPointSuccess) { fprintf(stderr, "driver entry point %s not found\n", name); exit(1); }
    };
    get("cuMemCreate", (void**)&create);
    get("cuMemRelease", (void**)&release);
    get("cuMemAddressReserve", (void**)&reserve);
    get("cuMemAddressFree", (void**)&free_range);
    get("cuMemMap", (void**)&map);
    get("cuMemUnmap", (void**)&unmap);
    get("cuMemSetAccess", (void**)&set_access);
    get("cuMemGetAllocationGranularity", (void**)&granularity);
    get("cuMemGetAllocationPropertiesFromHandle", (void**)&props);
    get("cuDeviceGetAttribute", (void**)&attribute);
  }
};

int main(int argc, char** argv) {
  const char* usage = "usage: %s <r1|r2|r3|r3lds> [--ctas-per-sm N] [--stages N] [--reps N] [--warmup N] [--alloc plain|compressible] "
                      "[--fill const|random|q1|q1:<column>]\n";
  if (argc < 2) { fprintf(stderr, usage, argv[0]); return 2; }
  const std::string variant = argv[1];
  int ctas_per_sm = variant == "r1" ? 4 : variant == "r2" ? 4 : 1, nstages = 3, reps = 30, warmup = 60;
  std::string alloc = "plain", fill = "const";
  for (int i = 2; i + 1 < argc; i += 2) {
    const std::string k = argv[i];
    const int v = atoi(argv[i + 1]);
    if (k == "--ctas-per-sm") ctas_per_sm = v;
    else if (k == "--stages") nstages = v;
    else if (k == "--reps") reps = v;
    else if (k == "--warmup") warmup = v;
    else if (k == "--alloc") alloc = argv[i + 1];
    else if (k == "--fill") fill = argv[i + 1];
    else { fprintf(stderr, "unknown option %s\n", k.c_str()); return 2; }
  }
  if (variant != "r1" && variant != "r2" && variant != "r3" && variant != "r3lds") { fprintf(stderr, "unknown variant %s\n", variant.c_str()); return 2; }
  if (nstages < 2 || nstages > MAX_STAGES || reps < 1) { fprintf(stderr, "bad --stages / --reps\n"); return 2; }
  if (alloc != "plain" && alloc != "compressible") { fprintf(stderr, "unknown --alloc %s\n", alloc.c_str()); return 2; }
  int q1_mask = -1;   // -1: not a q1 fill
  if (fill == "q1") q1_mask = (1 << NC) - 1;
  else if (fill.rfind("q1:", 0) == 0) {
    for (int c = 0; c < NC; c++) if (fill.substr(3) == COLUMN_NAMES[c]) q1_mask = 1 << c;
    if (q1_mask < 0) { fprintf(stderr, "unknown column in --fill %s\n", fill.c_str()); return 2; }
  } else if (fill != "const" && fill != "random") { fprintf(stderr, "unknown --fill %s\n", fill.c_str()); return 2; }

  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  const int sms = prop.multiProcessorCount;
  CK(cudaFree(nullptr));   // create the context before any driver call

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
  size_t span = slab_base + off + 4096;
  uint8_t* d = nullptr;
  int comp_supported = -1, chunks = 0, chunks_compressed = 0;
  size_t gran = 0, chunk_bytes = 0;
  Vmm vmm{};
  std::vector<CUmemGenericAllocationHandle> handles;
  CUdeviceptr range = 0;
  if (alloc == "plain") {
    CK(cudaMalloc(&d, span));
  } else {
    vmm.load();
    CUdevice dev = 0;
    CU(vmm.attribute(&comp_supported, CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED, dev));
    CUmemAllocationProp ap = {};
    ap.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    ap.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    ap.location.id = dev;
    ap.allocFlags.compressionType = CU_MEM_ALLOCATION_COMP_GENERIC;
    CU(vmm.granularity(&gran, &ap, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
    chunk_bytes = (SLAB + gran - 1) / gran * gran;
    span = (span + chunk_bytes - 1) / chunk_bytes * chunk_bytes;
    CU(vmm.reserve(&range, span, chunk_bytes, 0, 0));
    for (size_t o = 0; o < span; o += chunk_bytes) {
      CUmemGenericAllocationHandle h;
      CU(vmm.create(&h, chunk_bytes, &ap, 0));
      CUmemAllocationProp got = {};
      CU(vmm.props(&got, h));
      chunks++;
      chunks_compressed += got.allocFlags.compressionType == CU_MEM_ALLOCATION_COMP_GENERIC;
      CU(vmm.map(range + o, chunk_bytes, 0, h, 0));
      handles.push_back(h);
    }
    CUmemAccessDesc acc = {};
    acc.location = ap.location;
    acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    CU(vmm.set_access(range, span, &acc, 1));
    d = reinterpret_cast<uint8_t*>(range);
  }
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
  if (fill == "const") CK(cudaMemset(d, 0x5a, span));
  else if (fill == "random") random_fill_kernel<<<sms * 8, 256>>>(reinterpret_cast<uint64_t*>(d), (int64_t)(span / 8));
  else {
    CK(cudaMemset(d, 0, span));   // headers, alignment gaps and tail padding stay zero, as an arena slab's unwritten bytes
    q1_fill_kernel<<<sms * 8, 256>>>(d_batches, q1_mask, 1);
  }
  CK(cudaGetLastError());
  CK(cudaDeviceSynchronize());
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
  printf("{\"alloc\": \"%s\", \"fill\": \"%s\", \"compression_supported\": %d, \"granularity\": %zu, \"chunk_bytes\": %zu, "
         "\"chunks\": %d, \"chunks_compressed\": %d, ", alloc.c_str(), fill.c_str(), comp_supported, gran, chunk_bytes, chunks, chunks_compressed);
  printf("\"variant\": \"%s\", \"grid\": %d, \"threads\": %d, \"stages\": %d, \"stage_bytes\": %d, \"smem\": %zu, \"bytes\": %lld, "
         "\"reps\": %d, \"ms_median\": %.4f, \"ms_min\": %.4f, \"ms_max\": %.4f, \"gbps_median\": %.1f, \"gbps_best\": %.1f, \"check\": %u}\n",
         variant.c_str(), variant.rfind("r3", 0) == 0 ? sms : grid, variant == "r1" ? 512 : variant == "r2" ? THREADS : THREADS + 32,
         variant.rfind("r3", 0) == 0 ? nstages : 0, STAGE_BYTES, smem, (long long)algo, reps, med, best, ms[reps - 1],
         algo / (med * 1e-3) / 1e9, algo / (best * 1e-3) / 1e9, h_out);
  for (auto& e : ev) cudaEventDestroy(e);
  if (alloc == "plain") cudaFree(d);
  else {
    CU(vmm.unmap(range, span));
    for (auto h : handles) CU(vmm.release(h));
    CU(vmm.free_range(range, span));
  }
  cudaFree(d_batches);
  cudaFree(d_prefix);
  cudaFree(d_out);
  return 0;
}
