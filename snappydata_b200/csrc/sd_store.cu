// sd_store.cu -- device-resident ColumnBatch store: header/dictionary parsing on the host (the
// per-batch, per-column "decoder initialisation" the reference does in ColumnEncoding.getColumnDecoder
// / initializeNulls / initializeCursor, enc/ColumnEncoding.scala:797-832,1042-1099,
// enc/DictionaryEncoding.scala:85-116) and placement of the raw encoded bytes in HBM.
//
// HBM layout: the encoded bytes are copied VERBATIM (no re-encoding); only their placement is chosen
// by the engine: every buffer is positioned so that its first value / first dictionary index is
// 128-byte aligned, which makes every vector load of the scan kernel naturally aligned.  Null words get
// an 8-byte aligned side copy plus a host-computed "nulls before" prefix (one int32 per 512 rows).
#include <cuda.h>
#include <cudaTypedefs.h>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "sd_host.h"

namespace sd {

static thread_local std::string g_error;
int set_error(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_error = buf;
  return code;
}
const char* last_error_cstr() { return g_error.c_str(); }

std::vector<KernelEntry>& kernel_registry() {
  static std::vector<KernelEntry> r;
  return r;
}
std::string plan_struct_name(const std::string& signature) {
  unsigned long long h = 1469598103934665603ull;
  for (unsigned char ch : signature) { h ^= ch; h *= 1099511628211ull; }
  char b[40];
  snprintf(b, sizeof(b), "Plan_%016llx", h);
  return b;
}
AotRegistrar::AotRegistrar(const char* signature, const void* func, size_t tile_smem, int staged, size_t stage_bytes, const void* func2) {
  KernelEntry e;
  e.signature = signature; e.func = func; e.drv_func = nullptr; e.func2 = func2; e.tile_smem = (tile_smem + 15) & ~size_t(15); e.origin = "aot";
  e.staged = staged; e.stage_bytes = stage_bytes; e.name = plan_struct_name(e.signature);
  kernel_registry().push_back(e);
}

// ---- arena ------------------------------------------------------------------------------------------
// the driver's virtual memory calls, resolved through the runtime (the library does not link libcuda)
namespace {
struct Vmm {
  PFN_cuDeviceGet_v2000 device_get = nullptr;
  PFN_cuDeviceGetAttribute_v2000 attribute = nullptr;
  PFN_cuMemGetAllocationGranularity_v10020 granularity = nullptr;
  PFN_cuMemCreate_v10020 create = nullptr;
  PFN_cuMemGetAllocationPropertiesFromHandle_v10020 props = nullptr;
  PFN_cuMemAddressReserve_v10020 reserve = nullptr;
  PFN_cuMemMap_v10020 map = nullptr;
  PFN_cuMemSetAccess_v10020 set_access = nullptr;
  PFN_cuMemUnmap_v10020 unmap = nullptr;
  PFN_cuMemRelease_v10020 release = nullptr;
  PFN_cuMemAddressFree_v10020 address_free = nullptr;
  bool ok = false;
};
const Vmm& vmm() {
  static const Vmm v = [] {
    Vmm t;
    auto get = [](const char* name, void** fn) {
      cudaDriverEntryPointQueryResult q;
      return cudaGetDriverEntryPointByVersion(name, fn, 12000, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess;
    };
    t.ok = get("cuDeviceGet", (void**)&t.device_get) && get("cuDeviceGetAttribute", (void**)&t.attribute) &&
           get("cuMemGetAllocationGranularity", (void**)&t.granularity) && get("cuMemCreate", (void**)&t.create) &&
           get("cuMemGetAllocationPropertiesFromHandle", (void**)&t.props) && get("cuMemAddressReserve", (void**)&t.reserve) &&
           get("cuMemMap", (void**)&t.map) && get("cuMemSetAccess", (void**)&t.set_access) && get("cuMemUnmap", (void**)&t.unmap) &&
           get("cuMemRelease", (void**)&t.release) && get("cuMemAddressFree", (void**)&t.address_free);
    return t;
  }();
  return v;
}
#define SD_CU(call, what)                                                                        \
  do {                                                                                         \
    CUresult r__ = (call);                                                                     \
    if (r__ != CUDA_SUCCESS) { set_error(SD_ERR_CUDA, "%s failed: CUresult %d", what, (int)r__); goto fail; } \
  } while (0)

// 1: the device compresses generic allocations (*gran: their granularity); 0: it does not; < 0: error set
int compression_granularity(int device, size_t* gran) {
  const Vmm& v = vmm();
  if (!v.ok) return set_error(SD_ERR_CUDA, "the CUDA driver lacks the virtual memory entry points");
  CUdevice dev;
  int supported = 0;
  CUmemAllocationProp prop = {};
  if (v.device_get(&dev, device) != CUDA_SUCCESS ||
      v.attribute(&supported, CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED, dev) != CUDA_SUCCESS)
    return set_error(SD_ERR_CUDA, "device %d: compression support query failed", device);
  if (!supported) return 0;
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = dev;
  prop.allocFlags.compressionType = CU_MEM_ALLOCATION_COMP_GENERIC;
  if (v.granularity(gran, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED) != CUDA_SUCCESS)
    return set_error(SD_ERR_CUDA, "device %d: compressible allocation granularity query failed", device);
  return 1;
}

// a compressible slab of at least `want` bytes; false: error set, nothing held
bool vmm_slab(int device, size_t want, size_t gran, Arena::Slab* out) {
  const Vmm& v = vmm();
  const size_t sz = (want + gran - 1) / gran * gran;
  CUmemAllocationProp prop = {}, got = {};
  CUmemGenericAllocationHandle h = 0;
  CUdeviceptr va = 0;
  CUmemAccessDesc access = {};
  bool created = false, mapped = false;
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = device;
  prop.allocFlags.compressionType = CU_MEM_ALLOCATION_COMP_GENERIC;
  SD_CU(v.create(&h, sz, &prop, 0), "cuMemCreate");
  created = true;
  SD_CU(v.props(&got, h), "cuMemGetAllocationPropertiesFromHandle");
  SD_CU(v.reserve(&va, sz, gran, 0, 0), "cuMemAddressReserve");
  SD_CU(v.map(va, sz, 0, h, 0), "cuMemMap");
  mapped = true;
  access.location = prop.location;
  access.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  SD_CU(v.set_access(va, sz, &access, 1), "cuMemSetAccess");
  *out = {reinterpret_cast<uint8_t*>(va), sz, true, got.allocFlags.compressionType == CU_MEM_ALLOCATION_COMP_GENERIC, h};
  return true;
fail:
  if (mapped) v.unmap(va, sz);
  if (va) v.address_free(va, sz);
  if (created) v.release(h);
  return false;
}
}  // namespace

uint8_t* Arena::alloc(size_t n, size_t align, size_t misalign) {
  if (n == 0) n = 1;
  for (;;) {
    if (cur_slab < slabs.size()) {
      uint8_t* base = slabs[cur_slab].base;
      size_t p = (size_t)(uintptr_t)(base + cur_off);
      size_t want = (p + misalign + align - 1) / align * align - misalign;
      if (want < p) want += align;
      size_t off = want - (size_t)(uintptr_t)base;
      if (off + n <= slabs[cur_slab].bytes) {
        cur_off = off + n;
        used += n;
        slabs[cur_slab].used += n;
        if (record) record->push_back(Extent{base + off, n});
        return base + off;
      }
      cur_slab++;
      cur_off = 0;
      continue;
    }
    size_t sz = slab_bytes;
    if (n + align + misalign + 256 > sz) sz = n + align + misalign + 256;
    cudaSetDevice(device);
    size_t gran = 0;
    const int comp = compressible ? compression_granularity(device, &gran) : 0;
    if (comp < 0) return nullptr;
    if (comp) {
      Slab sl;
      if (!vmm_slab(device, sz, gran, &sl)) return nullptr;
      slabs.push_back(sl);
    } else {
      void* p = nullptr;
      cudaError_t e = cudaMalloc(&p, sz);
      if (e != cudaSuccess) {
        set_error(SD_ERR_CUDA, "cudaMalloc(%zu) failed: %s", sz, cudaGetErrorString(e));
        return nullptr;
      }
      slabs.push_back({(uint8_t*)p, sz, false, false, 0, 0});
    }
    cur_slab = slabs.size() - 1;
    cur_off = 0;
  }
}
void Arena::reset() {
  cur_slab = 0; cur_off = 0; used = 0;
  for (auto& s : slabs) s.used = 0;
}
Arena::Slab Arena::detach_slab(size_t i) {
  const Slab s = slabs[i];
  used -= s.used;
  slabs.erase(slabs.begin() + (ptrdiff_t)i);
  if (cur_slab > i) cur_slab--;
  else if (cur_slab == i) cur_off = 0;   // (the slab being allocated from: the next allocation moves on)
  return s;
}
void Arena::free_slab(int device, const Slab& s) {
  cudaSetDevice(device);
  if (s.vmm) {
    const Vmm& v = vmm();
    const CUdeviceptr va = reinterpret_cast<CUdeviceptr>(s.base);
    v.unmap(va, s.bytes);
    v.release(s.handle);
    v.address_free(va, s.bytes);
  } else {
    cudaFree(s.base);
  }
}
void Arena::release() {
  for (auto& s : slabs) free_slab(device, s);
  slabs.clear();
  reset();
}

uint8_t* PinnedArena::alloc(size_t n) {
  n = (n + 15) & ~size_t(15);
  if (n == 0) n = 16;
  for (;;) {
    if (cur_slab < slabs.size()) {
      if (cur_off + n <= slabs[cur_slab].second) { uint8_t* p = slabs[cur_slab].first + cur_off; cur_off += n; return p; }
      cur_slab++;
      cur_off = 0;
      continue;
    }
    const size_t sz = n > slab_bytes ? n : slab_bytes;
    void* p = nullptr;
    cudaError_t e = cudaHostAlloc(&p, sz, cudaHostAllocDefault);
    if (e != cudaSuccess) { set_error(SD_ERR_CUDA, "cudaHostAlloc(%zu) failed: %s", sz, cudaGetErrorString(e)); return nullptr; }
    slabs.emplace_back(reinterpret_cast<uint8_t*>(p), sz);
  }
}
PinnedArena::~PinnedArena() { for (auto& s : slabs) cudaFreeHost(s.first); }

// ---- little-endian host reads ----------------------------------------------------------------------
static inline int32_t rd_i32(const uint8_t* p) { int32_t v; memcpy(&v, p, 4); return v; }
static inline uint64_t rd_u64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }

static int fixed_width_of(int t) {
  switch (t) {
    case SD_BOOLEAN: case SD_BYTE: return 1;
    case SD_SHORT: return 2;
    case SD_INT: case SD_DATE: case SD_FLOAT: return 4;
    case SD_LONG: case SD_TIMESTAMP: case SD_DECIMAL: case SD_DOUBLE: return 8;
  }
  return 0;
}

template <class T>
static int upload_vec(sd_store* s, const std::vector<T>& v, size_t align, const T** out) {
  uint8_t* d = s->arena.alloc(v.size() * sizeof(T) + 16, align);
  if (!d) return SD_ERR_CUDA;
  if (!v.empty()) SD_CUDA(cudaMemcpyAsync(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, s->copy_stream));
  s->h2d_bytes += (int64_t)(v.size() * sizeof(T));
  *out = reinterpret_cast<const T*>(d);
  return 0;
}
static int upload_bytes(sd_store* s, const uint8_t* src, size_t n, size_t align, size_t misalign, uint8_t** out) {
  uint8_t* d = s->arena.alloc(n + 160, align, misalign);   // tail padding: vector loads may overrun a partial pair
  if (!d) return SD_ERR_CUDA;
  cudaStream_t st = s->copy_stream;
  if (s->num_copy_streams > 1 && n >= (size_t(64) << 10)) {   // big buffers rotate over several H2D streams
    const int k = s->next_stream++ % s->num_copy_streams;
    if (k > 0) st = s->extra_streams[k - 1];
  }
  if (n) SD_CUDA(cudaMemcpyAsync(d, src, n, cudaMemcpyHostToDevice, st));
  s->h2d_bytes += (int64_t)n;
  *out = d;
  return 0;
}

// Parse [numElements][dictionary] at p; returns bytes consumed or -1.
static int64_t parse_dictionary(const uint8_t* p, const uint8_t* end, int type, int* n_out, std::vector<std::string>* strings,
                                std::vector<int64_t>* rec_off = nullptr, const uint8_t* buf0 = nullptr) {
  if (p + 4 > end) return -1;
  const int n = rd_i32(p);
  if (n < 0) return -1;
  const uint8_t* q = p + 4;
  if (type == SD_STRING) {
    strings->clear();
    strings->reserve(n);
    for (int k = 0; k < n; k++) {
      if (q + 4 > end) return -1;
      const int l = rd_i32(q);
      if (l < 0 || q + 4 + l > end) return -1;
      strings->emplace_back(reinterpret_cast<const char*>(q + 4), (size_t)l);
      if (rec_off) rec_off->push_back(q - buf0);
      q += 4 + l;
    }
  } else if (type == SD_INT || type == SD_DATE) {
    q += 4 * (int64_t)n;
  } else if (type == SD_LONG || type == SD_TIMESTAMP) {
    q += 8 * (int64_t)n;   // written 8 bytes per entry (allocation slack stays at the tail)
  } else return -2;
  if (q > end) return -1;
  *n_out = n;
  return q - p;
}

// device_fill_total >= 0: `buf` holds only the buffer's prefix (header, null words, dictionary) and a kernel of the caller
// writes the whole buffer (device_fill_total bytes) at the device address this function reserves (sd_encode.cu)
// wide: a DECIMAL column of more than 18 digits (variable-width records, laid out like a raw STRING body)
static int upload_column(sd_store* s, const uint8_t* buf, int64_t len, int type, int nullable, int num_rows, StoredCol& c,
                         int64_t device_fill_total = -1, bool wide = false) {
  if (len < 8) return set_error(SD_ERR_INVALID, "column buffer shorter than its 8-byte header");
  const bool device_fill = device_fill_total >= 0;
  if (device_fill) len = device_fill_total;
  // ---- compressed envelope [-codecId][uncompressedLen][payload] (CompressionUtils.scala:53-61): only the
  //      compressed bytes go to the device; the host decodes just the leading bytes it must parse -------
  const uint8_t* payload = nullptr;
  int64_t payload_len = 0;
  std::vector<uint8_t> prefix;
  std::vector<uint8_t> host_full;   // whole buffer decompressed on the host (Snappy; LZ4 of encodings that need a host walk)
  if (rd_i32(buf) < 0 && -rd_i32(buf) != 1) {
    // Snappy (the reference's non-default codec): decompressed on the host like the reference's iterator does
    // (ColumnBatchIterator.scala:102-113), then handled as an uncompressed buffer
    int rc0 = decompress_envelope_host(buf, len, host_full);
    if (rc0) return rc0;
    buf = host_full.data();
    len = (int64_t)host_full.size();
    if (len < 8) return set_error(SD_ERR_INVALID, "column buffer shorter than its 8-byte header");
  }
  if (rd_i32(buf) < 0) {
    const int64_t ulen = rd_i32(buf + 4);
    if (ulen < 8) return set_error(SD_ERR_INVALID, "compressed column buffer: bad uncompressed length %lld", (long long)ulen);
    payload = buf + 8;
    payload_len = len - 8;
    int64_t want = 8;
    for (;;) {
      want = std::min(want, ulen);
      prefix.assign((size_t)want + 16, 0);
      const int64_t got = lz4_decode_prefix(payload, payload_len, prefix.data(), want);
      if (got < want) return set_error(SD_ERR_INVALID, "corrupt LZ4 column buffer");
      const int tid = rd_i32(prefix.data());
      const int nb = want >= 8 ? rd_i32(prefix.data() + 4) : 0;
      if (tid < 0 || tid > ENC_BOOLEAN_BITSET || nb < 0 || (nb & 7) || 8 + (int64_t)nb > ulen) return set_error(SD_ERR_INVALID, "corrupt header in LZ4 column buffer");
      int64_t need = 8 + nb;
      // encodings whose layout needs a host walk over every value (run lengths, variable-width strings): decode it all here
      if (tid == ENC_RUN_LENGTH || (tid == ENC_UNCOMPRESSED && (type == SD_STRING || wide))) need = ulen;
      if (tid == ENC_DICTIONARY || tid == ENC_BIG_DICTIONARY) {
        need += 4;
        if (want >= need) {
          const int n = rd_i32(prefix.data() + 8 + nb);
          if (n < 0) return set_error(SD_ERR_INVALID, "corrupt dictionary in LZ4 column buffer");
          if (type == SD_INT || type == SD_DATE) need += 4 * (int64_t)n;
          else if (type == SD_LONG || type == SD_TIMESTAMP) need += 8 * (int64_t)n;
          else {   // strings: walk what we have; ask for more when the walk runs off the decoded prefix
            int64_t q = 8 + nb + 4;
            bool short_prefix = false;
            for (int k = 0; k < n; k++) {
              if (q + 4 > want) { short_prefix = true; break; }
              const int l = rd_i32(prefix.data() + q);
              if (l < 0) return set_error(SD_ERR_INVALID, "corrupt string dictionary in LZ4 column buffer");
              q += 4 + l;
            }
            need = short_prefix || q > want ? std::max<int64_t>(q, want * 2) : q;
          }
        }
      }
      need = std::min(need, ulen);
      if (want >= need) break;
      want = need;
    }
    buf = prefix.data();
    len = ulen;
    if (want >= ulen) payload = nullptr;   // fully decoded on the host: uploaded as plain bytes, nothing left for the device decoder
  }
  const int type_id = rd_i32(buf);
  if (type_id > ENC_BOOLEAN_BITSET) return set_error(SD_ERR_INVALID, "unknown encoding typeId %d", type_id);
  const int null_bytes = rd_i32(buf + 4);
  if (null_bytes < 0 || (null_bytes & 7) || 8 + (int64_t)null_bytes > len) return set_error(SD_ERR_INVALID, "bad null bitset size %d", null_bytes);
  if (!nullable && null_bytes != 0)   // NotNullDecoder.initializeNulls (enc/ColumnEncoding.scala:1042-1050)
    return set_error(SD_ERR_INVALID, "Nulls bitset of size %d found in NOT NULL column", null_bytes);
  const int nwords = null_bytes >> 3;
  c = StoredCol();
  c.present = true;
  c.len = len;
  memset(&c.dev, 0, sizeof(c.dev));
  c.dev.enc = type_id;
  c.dev.nwords = nwords;
  // nulls before each tile (the incremental numNulls bookkeeping of the generated loop,
  // ColumnTableScan.scala:794-815, turned into a prefix the kernel can index)
  const int ntiles = (num_rows + NULL_PREFIX_ROWS - 1) / NULL_PREFIX_ROWS;
  int64_t total_nulls = 0;
  std::vector<int32_t> tile_nulls;
  if (nwords) {
    tile_nulls.resize((ntiles > 0 ? ntiles : 1) + 1, 0);
    for (int w = 0; w < nwords; w++) {
      if ((w % NULL_PREFIX_WORDS) == 0 && w / NULL_PREFIX_WORDS < ntiles) tile_nulls[w / NULL_PREFIX_WORDS] = (int32_t)total_nulls;
      uint64_t word = rd_u64(buf + 8 + 8 * (int64_t)w);
      if ((int64_t)(w + 1) * 64 > num_rows) {   // ignore bits beyond the batch
        int valid = num_rows - w * 64;
        word = valid <= 0 ? 0 : (valid >= 64 ? word : (word & ((1ull << valid) - 1)));
      }
      total_nulls += __builtin_popcountll(word);
    }
    for (int t = (nwords + NULL_PREFIX_WORDS - 1) / NULL_PREFIX_WORDS; t < ntiles; t++) tile_nulls[t] = (int32_t)total_nulls;
    tile_nulls.back() = (int32_t)total_nulls;
  }
  c.has_nulls = nwords > 0;
  const int64_t nn = num_rows - total_nulls;   // stored (non-null) values
  const uint8_t* end = buf + len;
  int64_t body = 8 + null_bytes;
  int64_t dict_bytes = 0;
  const int w = fixed_width_of(type);
  std::vector<int32_t> run_ends, run_codes, str_pos;
  switch (type_id) {
    case ENC_UNCOMPRESSED:
      if (wide) {
        // DECIMAL(p > 18): back-to-back [len:int32][unscaled value, BigInteger.toByteArray] (enc/Uncompressed.scala:330-345),
        // walked like a raw STRING body; a value of precision <= 38 takes 1..16 bytes
        const uint8_t* q = buf + body;
        str_pos.reserve((size_t)nn);
        for (int64_t k = 0; k < nn; k++) {
          if (q + 4 > end) return set_error(SD_ERR_INVALID, "uncompressed DECIMAL column truncated at value %lld", (long long)k);
          const int32_t l = rd_i32(q);
          if (l < 1 || l > 16 || q + 4 + l > end)
            return set_error(SD_ERR_INVALID, "uncompressed DECIMAL column: value %lld has %d bytes (1..16 expected)", (long long)k, l);
          if (q - (buf + body) > INT32_MAX) return set_error(SD_ERR_UNSUPPORTED, "uncompressed DECIMAL body beyond 2 GB");
          str_pos.push_back((int32_t)(q - (buf + body)));
          q += 4 + l;
        }
        c.raw_str = true;
        break;
      }
      if (type == SD_STRING) {
        // variable width: back-to-back [len:int32][bytes]; the reference reads it with a sequential cursor
        // (enc/Uncompressed.scala:116-161).  One host walk per buffer gives every stored value's record position, which
        // the kernel then loads like a 4-byte column; the bytes themselves stay where they are.
        const uint8_t* q = buf + body;
        str_pos.reserve((size_t)nn);
        for (int64_t k = 0; k < nn; k++) {
          if (q + 4 > end) return set_error(SD_ERR_INVALID, "uncompressed STRING column truncated at value %lld", (long long)k);
          const int32_t l = rd_i32(q);
          if (l < 0 || q + 4 + l > end) return set_error(SD_ERR_INVALID, "uncompressed STRING column: bad length %d at value %lld", l, (long long)k);
          if (q - (buf + body) > INT32_MAX) return set_error(SD_ERR_UNSUPPORTED, "uncompressed STRING body beyond 2 GB");
          str_pos.push_back((int32_t)(q - (buf + body)));
          q += 4 + l;
        }
        c.raw_str = true;
        break;
      }
      if (body + nn * w > len) return set_error(SD_ERR_INVALID, "uncompressed column truncated: need %lld bytes, have %lld", (long long)(body + nn * w), (long long)len);
      break;
    case ENC_DICTIONARY: case ENC_BIG_DICTIONARY: {
      int n = 0;
      int64_t used = parse_dictionary(buf + body, end, type, &n, &c.dict_strings, &c.dict_rec_off, buf);
      if (used == -2) return set_error(SD_ERR_INVALID, "DictionaryDecoder not supported for sd_type %d", type);
      if (used < 0) return set_error(SD_ERR_INVALID, "truncated dictionary");
      dict_bytes = used;
      c.dev.dict_n = n;
      body += used;
      const int iw = type_id == ENC_DICTIONARY ? 2 : 4;
      if (body + nn * iw > len) return set_error(SD_ERR_INVALID, "dictionary indexes truncated");
      break;
    }
    case ENC_BOOLEAN_BITSET:
      if (type != SD_BOOLEAN) return set_error(SD_ERR_INVALID, "BooleanBitSet encoding on a non-boolean column");
      if (body + ((nn + 63) / 64) * 8 > len) return set_error(SD_ERR_INVALID, "boolean bitset truncated");
      break;
    case ENC_RUN_LENGTH: {
      if (type == SD_BYTE || type == SD_BOOLEAN)
        return set_error(SD_ERR_UNSUPPORTED, "RunLength BYTE/BOOLEAN: the reference decoder is inconsistent (enc/RunLengthEncoding.scala:99-110)");
      if (!(type == SD_SHORT || type == SD_INT || type == SD_DATE || type == SD_LONG || type == SD_TIMESTAMP || type == SD_STRING))
        return set_error(SD_ERR_INVALID, "RunLengthDecoder not supported for sd_type %d", type);
      const uint8_t* q = buf + body;
      int64_t covered = 0;
      std::unordered_map<std::string, int> seen;
      while (covered < nn) {
        if (type == SD_STRING) {
          if (q + 4 > end) return set_error(SD_ERR_INVALID, "RunLengthEncoding: reading next run after data end");
          int l = rd_i32(q);
          if (l < 0 || q + 8 + l > end) return set_error(SD_ERR_INVALID, "RunLengthEncoding: truncated string run");
          std::string sv(reinterpret_cast<const char*>(q + 4), (size_t)l);
          auto it = seen.find(sv);
          int code;
          if (it == seen.end()) { code = (int)c.dict_strings.size(); seen.emplace(sv, code); c.dict_strings.push_back(sv); c.dict_rec_off.push_back(q - buf); } else code = it->second;
          run_codes.push_back(code);
          covered += rd_i32(q + 4 + l);
          q += 8 + l;
        } else {
          if (q + w + 4 > end) return set_error(SD_ERR_INVALID, "RunLengthEncoding: reading next run after data end");
          covered += rd_i32(q + w);
          q += w + 4;
        }
        if (covered > INT32_MAX) return set_error(SD_ERR_INVALID, "run lengths overflow");
        run_ends.push_back((int32_t)covered);
      }
      c.dev.nruns = (int)run_ends.size();
      if (type == SD_STRING) c.dev.dict_n = (int)c.dict_strings.size();
      break;
    }
  }
  c.body_off = body;
  c.algo_bytes = len - 8 - dict_bytes;
  if (!c.unsupported.empty()) return 0;   // recorded; an error only if a plan scans this column

  int rc = 0;
  if (payload) {   // expanded on the device at the next flush: [dev_base, dev_base + len) is written by the LZ4 kernel
    c.dev_base = s->arena.alloc((size_t)len + 160, 128, (size_t)body);
    uint8_t* d_src = nullptr;
    if (s->span_h0 && payload >= s->span_h0 && payload + payload_len <= s->span_h0 + s->span_len) {
      d_src = s->span_d0 + (payload - s->span_h0);   // already on its way with the batch's span copy
      if (!c.dev_base) return SD_ERR_CUDA;
    } else {
      d_src = s->lz4_stage.alloc((size_t)payload_len + 32, 16);
      if (!c.dev_base || !d_src) return SD_ERR_CUDA;
      SD_CUDA(cudaMemcpyAsync(d_src, payload, (size_t)payload_len, cudaMemcpyHostToDevice, s->copy_stream));
      s->h2d_bytes += payload_len;
    }
    s->pending_lz4.push_back(Lz4Job{d_src, c.dev_base, payload_len, len});
    s->lz4_buffers++; s->lz4_in_bytes += payload_len; s->lz4_out_bytes += len;
  } else if (device_fill) {
    c.dev_base = s->arena.alloc((size_t)len + 160, 128, (size_t)body);
    if (!c.dev_base) return SD_ERR_CUDA;
  } else {
    rc = upload_bytes(s, buf, (size_t)len, 128, (size_t)body, &c.dev_base);
    if (rc) return rc;
  }
  c.dev.data = c.dev_base + body;
  if (c.raw_str) {   // the kernel's view: positions as the column's data, the body as its "dictionary"
    const int32_t* dp = nullptr;
    str_pos.resize(str_pos.size() + 40, 0);   // tail padding: vector loads may overrun a partial pair
    rc = upload_vec(s, str_pos, 128, &dp);     // (pageable source: staged before the call returns)
    if (rc) return rc;
    c.dev.dict = c.dev_base + body;
    c.dev.data = reinterpret_cast<const uint8_t*>(dp);
    c.dev.enc = ENC_STR_RAW;
    c.dev.dict_n = 0;
  }
  if ((type_id == ENC_DICTIONARY || type_id == ENC_BIG_DICTIONARY) && type != SD_STRING) {
    const int ew = (type == SD_INT || type == SD_DATE) ? 4 : 8;
    c.dev.dict = c.dev_base + body - (int64_t)ew * c.dev.dict_n;   // ew-aligned because `body` is 128-aligned
  }
  if (nwords) {
    uint8_t* dn = nullptr;
    rc = upload_bytes(s, buf + 8, (size_t)null_bytes, 8, 0, &dn);
    if (rc) return rc;
    c.dev.nulls = reinterpret_cast<const uint64_t*>(dn);
    rc = upload_vec(s, tile_nulls, 4, &c.dev.tile_nulls);
    if (rc) return rc;
  }
  if (type_id == ENC_RUN_LENGTH) {
    rc = upload_vec(s, run_ends, 4, &c.dev.run_ends);
    if (rc) return rc;
    if (type == SD_STRING) {
      const int32_t* dc = nullptr;
      rc = upload_vec(s, run_codes, 4, &dc);
      if (rc) return rc;
      c.dev.dict = reinterpret_cast<const uint8_t*>(dc);
    }
  }
  const int kind = wide ? K_CODE : kind_of_type(type);
  c.fast = !c.has_nulls && ((kind == K_CODE && (type_id == ENC_DICTIONARY || type_id == ENC_BIG_DICTIONARY || c.raw_str)) ||
                            (kind != K_CODE && type_id == ENC_UNCOMPRESSED));
  // string values by reference (hash-table keys): device address of every dictionary entry's record
  if (type == SD_STRING && !c.raw_str) {
    c.dict_rec_ptr.assign(c.dict_strings.size(), 0);
    for (size_t k = 0; k < c.dict_strings.size() && k < c.dict_rec_off.size(); k++) c.dict_rec_ptr[k] = (int64_t)(uintptr_t)(c.dev_base + c.dict_rec_off[k]);
  }
  return 0;
}

// update delta: header + relative null words, [numBaseRows][numDeltas][positions], pad to 8, values
// (enc/ColumnDeltaEncoder.scala:300-331; decoder init enc/ColumnDeltaDecoder.scala:47-61)
static int upload_delta(sd_store* s, const uint8_t* buf, int64_t len, int type, StoredCol& col, int depth) {
  StoredDelta& d = col.delta[depth];
  std::vector<uint8_t> plain;
  if (len >= 8 && rd_i32(buf) < 0) {   // stored compressed (a depth-1 delta of ~1.3k doubles passes the 2048-byte threshold): small, host-side
    int rc0 = decompress_envelope_host(buf, len, plain);
    if (rc0) return rc0;
    buf = plain.data();
    len = (int64_t)plain.size();
  }
  if (len < 16) return set_error(SD_ERR_INVALID, "delta buffer too short");
  const int type_id = rd_i32(buf);
  if (type_id < 0) return set_error(SD_ERR_INVALID, "doubly compressed delta buffer");
  const int null_bytes = rd_i32(buf + 4);
  if (null_bytes < 0 || (null_bytes & 7) || 16 + (int64_t)null_bytes > len) return set_error(SD_ERR_INVALID, "bad delta null bitset size");
  const uint8_t* cpos = buf + 8 + null_bytes;
  const int n = rd_i32(cpos + 4);
  if (n < 0 || 16 + (int64_t)null_bytes + 4 * (int64_t)n > len) return set_error(SD_ERR_INVALID, "delta positions truncated");
  // the kernels index shared-memory bitmaps and delta values with these: they must be ascending ordinals of the base batch
  {
    const int nbase = rd_i32(cpos);
    int32_t prev = -1;
    for (int k = 0; k < n; k++) {
      const int32_t pos = rd_i32(cpos + 8 + 4 * (int64_t)k);
      if (pos <= prev || pos < 0 || (nbase > 0 && pos >= nbase)) return set_error(SD_ERR_INVALID, "delta positions must be ascending ordinals below %d (entry %d is %d)", nbase, k, pos);
      prev = pos;
    }
  }
  int64_t data_off = ((8 + null_bytes + 8 + 4 * (int64_t)n + 7) >> 3) << 3;   // round to nearest word
  d = StoredDelta();
  d.present = true;
  d.len = len;
  d.nbase = rd_i32(cpos);
  d.body_off = data_off;
  memset(&d.dev, 0, sizeof(d.dev));
  d.dev.n = n; d.dev.enc = type_id; d.dev.nwords = null_bytes >> 3;
  uint8_t* p = nullptr;
  int rc = upload_bytes(s, cpos + 8, 4 * (size_t)n, 16, 0, &p);
  if (rc) return rc;
  d.dev.positions = reinterpret_cast<const int32_t*>(p);
  if (null_bytes) {
    rc = upload_bytes(s, buf + 8, (size_t)null_bytes, 8, 0, &p);
    if (rc) return rc;
    d.dev.nulls = reinterpret_cast<const uint64_t*>(p);
  }
  const uint8_t* end = buf + len;
  int64_t body = data_off;
  if (type_id == ENC_DICTIONARY || type_id == ENC_BIG_DICTIONARY) {
    int dn = 0;
    int64_t used = parse_dictionary(buf + body, end, type, &dn, &d.dict_strings);
    if (used < 0) return set_error(SD_ERR_INVALID, "bad delta dictionary");
    d.dev.dict_n = dn;
    if (type != SD_STRING) {
      const int ew = (type == SD_INT || type == SD_DATE) ? 4 : 8;
      rc = upload_bytes(s, buf + body + 4, (size_t)ew * dn, 16, 0, &p);
      if (rc) return rc;
      d.dev.dict = p;
    }
    body += used;
  } else if (type_id == ENC_UNCOMPRESSED) {
    if (type == SD_STRING) { col.unsupported = "Uncompressed STRING update delta"; return 0; }
  } else if (type_id == ENC_BOOLEAN_BITSET) {
    if (type != SD_BOOLEAN) return set_error(SD_ERR_INVALID, "BooleanBitSet delta on a non-boolean column");
  } else return set_error(SD_ERR_UNSUPPORTED, "RunLength-encoded update delta");
  if (body > len) return set_error(SD_ERR_INVALID, "delta values truncated");
  {   // the value bytes must cover the non-null entries
    int64_t nulls = 0;
    for (int wd = 0; wd < (null_bytes >> 3); wd++) nulls += __builtin_popcountll(rd_u64(buf + 8 + 8 * (int64_t)wd));
    const int64_t nnv = n - nulls;
    int64_t need = 0;
    if (type_id == ENC_UNCOMPRESSED) need = nnv * fixed_width_of(type);
    else if (type_id == ENC_BOOLEAN_BITSET) need = ((nnv + 63) / 64) * 8;
    else need = nnv * (type_id == ENC_DICTIONARY ? 2 : 4);
    if (nnv < 0 || body + need > len) return set_error(SD_ERR_INVALID, "delta values truncated: %lld entries need %lld bytes, %lld present", (long long)nnv, (long long)need, (long long)(len - body));
  }
  rc = upload_bytes(s, buf + body, (size_t)(len - body), 16, 0, &p);
  if (rc) return rc;
  d.dev.data = p;
  return 0;
}

int store_install(sd_store* s, FreshBatches& fresh, const std::vector<const StoredBatch*>& remove, const char* what) {
  std::lock_guard<std::mutex> lock(s->mu);
  std::unordered_map<const StoredBatch*, size_t> where;
  for (size_t i = 0; i < s->batches.size(); i++) where.emplace(s->batches[i].get(), i);
  for (auto& f : fresh)
    if (!where.count(f.first)) return set_error(SD_ERR_STATE, "%s: a batch of the snapshot left the store", what);
  for (const StoredBatch* r : remove)
    if (!where.count(r)) return set_error(SD_ERR_STATE, "%s: a batch of the snapshot left the store", what);
  const int64_t v = s->version + 1;   // snapshots older than this one may still read what leaves the store now
  for (auto& f : fresh) {
    const size_t i = where[f.first];
    prune_extents(*f.second);
    s->batches[i]->retired_at = v;
    s->retired.push_back(std::move(s->batches[i]));
    s->batches[i] = std::move(f.second);
  }
  if (!remove.empty()) {
    std::vector<bool> drop(s->batches.size(), false);
    for (const StoredBatch* r : remove) drop[where[r]] = true;
    size_t k = 0;
    for (size_t i = 0; i < s->batches.size(); i++) {
      if (drop[i]) { s->batches[i]->retired_at = v; s->retired.push_back(std::move(s->batches[i])); }
      else s->batches[k++] = std::move(s->batches[i]);
    }
    s->batches.resize(k);
  }
  s->version = v;
  return 0;
}

void prune_extents(StoredBatch& b) {
  std::vector<Extent>& e = b.extents;
  std::sort(e.begin(), e.end(), [](const Extent& x, const Extent& y) { return x.ptr < y.ptr; });
  std::vector<char> used(e.size(), 0);
  visit_device_pointers(b, [&](uintptr_t a, int, const char*) {
    auto it = std::upper_bound(e.begin(), e.end(), a, [](uintptr_t x, const Extent& y) { return x < (uintptr_t)y.ptr; });
    if (it != e.begin() && a < (uintptr_t)(it - 1)->ptr + (it - 1)->bytes) used[(size_t)(it - e.begin() - 1)] = 1;
    return a;
  });
  size_t k = 0;
  for (size_t i = 0; i < e.size(); i++) if (used[i]) e[k++] = e[i];
  e.resize(k);
}

int store_register_encoded(sd_store* s, const uint8_t* prefix, int64_t prefix_len, int64_t total_len, int type, int nullable,
                           int num_rows, StoredCol& c) {
  if (total_len < prefix_len) return set_error(SD_ERR_INVALID, "encoded column shorter than its prefix");
  return upload_column(s, prefix, prefix_len, type, nullable, num_rows, c, total_len);
}

int store_flush_lz4(sd_store* s) {
  if (s->pending_lz4.empty()) return 0;
  SD_CUDA(cudaSetDevice(s->device));
  if (!s->d_lz4_error) {
    SD_CUDA(cudaMalloc(&s->d_lz4_error, 64));
    SD_CUDA(cudaMemset(s->d_lz4_error, 0, 64));
    SD_CUDA(cudaEventCreateWithFlags(&s->lz4_copied, cudaEventDisableTiming));
    for (int k = 0; k < sd_store::LZ4_STREAMS; k++) {
      SD_CUDA(cudaStreamCreateWithFlags(&s->lz4_streams[k], cudaStreamNonBlocking));
      SD_CUDA(cudaEventCreateWithFlags(&s->lz4_done[k], cudaEventDisableTiming));
    }
  }
  const size_t nbytes = s->pending_lz4.size() * sizeof(Lz4Job);
  uint8_t* d_jobs = s->lz4_stage.alloc(nbytes + 16, 16);
  if (!d_jobs) return SD_ERR_CUDA;
  uint8_t* h_jobs = s->lz4_jobs_host.alloc(nbytes);
  if (!h_jobs) return SD_ERR_CUDA;
  memcpy(h_jobs, s->pending_lz4.data(), nbytes);
  SD_CUDA(cudaMemcpyAsync(d_jobs, h_jobs, nbytes, cudaMemcpyHostToDevice, s->copy_stream));
  SD_CUDA(cudaEventRecord(s->lz4_copied, s->copy_stream));   // the compressed payloads went over this stream too
  int nstreams = sd_store::LZ4_STREAMS;
  if (const char* e = getenv("SD_TUNE_LZ4_STREAMS")) { const int v = atoi(e); if (v >= 1 && v <= sd_store::LZ4_STREAMS) nstreams = v; }
  const int k = s->lz4_next++ % nstreams;
  SD_CUDA(cudaStreamWaitEvent(s->lz4_streams[k], s->lz4_copied, 0));
  for (int q = 0; q + 1 < s->num_copy_streams; q++) {   // ... and over the extra copy queues
    SD_CUDA(cudaEventRecord(s->extra_done[q], s->extra_streams[q]));
    SD_CUDA(cudaStreamWaitEvent(s->lz4_streams[k], s->extra_done[q], 0));
  }
  int rc = lz4_launch(s->lz4_streams[k], reinterpret_cast<const Lz4Job*>(d_jobs), (int)s->pending_lz4.size(), s->d_lz4_error);
  if (rc) return rc;
  SD_CUDA(cudaEventRecord(s->lz4_done[k], s->lz4_streams[k]));
  s->lz4_used[k] = true;
  s->pending_lz4.clear();
  return 0;
}

int store_lz4_order(sd_store* s, cudaStream_t stream) {
  for (int k = 0; k < sd_store::LZ4_STREAMS; k++)
    if (s->lz4_used[k]) SD_CUDA(cudaStreamWaitEvent(stream, s->lz4_done[k], 0));
  return 0;
}

int store_lz4_check(sd_store* s) {
  bool any = false;
  for (int k = 0; k < sd_store::LZ4_STREAMS; k++) any = any || s->lz4_used[k];
  if (!any) return 0;
  SD_CUDA(cudaSetDevice(s->device));
  for (int k = 0; k < sd_store::LZ4_STREAMS; k++)
    if (s->lz4_used[k]) { SD_CUDA(cudaStreamSynchronize(s->lz4_streams[k])); s->lz4_used[k] = false; }
  unsigned int err = 0;
  SD_CUDA(cudaMemcpy(&err, s->d_lz4_error, 4, cudaMemcpyDeviceToHost));
  if (s->pending_lz4.empty()) { s->lz4_stage.reset(); s->lz4_jobs_host.reset(); }   // nothing refers to the staged payloads any more
  if (err) {
    SD_CUDA(cudaMemset(s->d_lz4_error, 0, 4));
    return set_error(SD_ERR_INVALID, "corrupt LZ4 payload in a column buffer (device decode failed)");
  }
  return 0;
}

int store_put(sd_store* s, const sd_batch* b, const int32_t* table_ordinals, bool images) {
  if (!b || b->num_rows < 0) return set_error(SD_ERR_INVALID, "bad batch");
  std::lock_guard<std::mutex> lock(s->mu);
  cudaSetDevice(s->device);
  std::unique_ptr<StoredBatch> sb(new StoredBatch());
  sb->num_rows = b->num_rows; sb->bucket_id = b->bucket_id; sb->batch_id = b->batch_id;
  sb->cols.resize(s->schema.size());
  ExtentRecorder rec(s->arena, &sb->extents);   // every arena allocation of this put belongs to the new batch
  const size_t lz4_before = s->pending_lz4.size();
  {   // LZ4 envelopes that lie (almost) back to back in host memory: one host->device copy for the lot (small copies reach
      // a lower link rate than large ones)
    s->span_h0 = nullptr;
    const uint8_t *lo = nullptr, *hi = nullptr;
    size_t sum = 0;
    int cnt = 0;
    for (int i = 0; i < b->ncols; i++) {
      const uint8_t* buf = reinterpret_cast<const uint8_t*>(b->col_bufs[i]);
      if (!buf || b->col_lens[i] < 16 || rd_i32(buf) != -1) continue;
      if (!lo || buf < lo) lo = buf;
      if (!hi || buf + b->col_lens[i] > hi) hi = buf + b->col_lens[i];
      sum += (size_t)b->col_lens[i];
      cnt++;
    }
    if (cnt >= 2 && (size_t)(hi - lo) <= sum + sum / 8 + 4096) {
      const size_t span = (size_t)(hi - lo);
      uint8_t* d0 = s->lz4_stage.alloc(span + 64, 16, (16 - (reinterpret_cast<uintptr_t>(lo) & 15)) & 15);   // same residue mod 16 as the host span
      if (!d0) return SD_ERR_CUDA;
      cudaStream_t st = s->copy_stream;
      if (s->num_copy_streams > 1) {   // SD_TUNE_COPY_STREAMS: span copies rotate over several H2D queues (a copy's setup hides under its neighbour)
        const int k = s->next_stream++ % s->num_copy_streams;
        if (k > 0) st = s->extra_streams[k - 1];
      }
      SD_CUDA(cudaMemcpyAsync(d0, lo, span, cudaMemcpyHostToDevice, st));
      s->h2d_bytes += (int64_t)span;
      s->span_h0 = lo; s->span_d0 = d0; s->span_len = span;
    }
  }
  for (int i = 0; i < b->ncols; i++) {
    const int t = table_ordinals ? table_ordinals[i] : i;
    if (t < 0 || t >= (int)s->schema.size()) return set_error(SD_ERR_INVALID, "table column %d outside the store schema", t);
    const uint8_t* buf = reinterpret_cast<const uint8_t*>(b->col_bufs[i]);
    if (!buf) continue;
    StoredCol& c = sb->cols[t];
    if (c.present) continue;   // same table column projected twice
    const bool wide = wide_decimal(s->schema[t].type, s->schema[t].precision);
    int rc = upload_column(s, buf, b->col_lens[i], s->schema[t].type, s->schema[t].nullable, b->num_rows, c, -1, wide);
    if (rc) return rc;
    for (int depth = 0; depth < 2; depth++) {
      const void* const* arr = depth == 0 ? b->delta0 : b->delta1;
      const int64_t* lens = depth == 0 ? b->delta0_lens : b->delta1_lens;
      if (arr && arr[i] && wide) {   // kept, like any delta the engine cannot decode: a scan of this column is refused
        c.unsupported = "update delta on a DECIMAL wider than 18 digits";
        sb->has_deltas = true;
        c.fast = false;
        continue;
      }
      if (arr && arr[i]) {
        rc = upload_delta(s, reinterpret_cast<const uint8_t*>(arr[i]), lens[i], s->schema[t].type, c, depth);
        if (rc) return rc;
        sb->has_deltas = true;
        c.fast = false;
      }
    }
    // unified code space of a STRING column: base dictionary [0,n), NULL = n, then delta-only strings;
    // delta dictionaries are translated to it so per-batch tables cover base and updated values alike
    if (s->schema[t].type == SD_STRING && (c.delta[0].present || c.delta[1].present)) {
      std::unordered_map<std::string, int> code;
      for (size_t k = 0; k < c.dict_strings.size(); k++) code.emplace(c.dict_strings[k], (int)k);
      const int base_n = c.dev.dict_n;
      std::vector<std::string> extra;
      for (int depth = 0; depth < 2; depth++) {
        StoredDelta& d = c.delta[depth];
        if (!d.present) continue;
        std::vector<int32_t> map(d.dict_strings.size());
        for (size_t k = 0; k < d.dict_strings.size(); k++) {
          auto it = code.find(d.dict_strings[k]);
          if (it == code.end()) {
            const int nc = base_n + 1 + (int)extra.size();
            extra.push_back(d.dict_strings[k]);
            code.emplace(d.dict_strings[k], nc);
            map[k] = nc;
          } else map[k] = it->second;
        }
        const int32_t* dm = nullptr;
        rc = upload_vec(s, map, 4, &dm);
        if (rc) return rc;
        d.dev.dict = reinterpret_cast<const uint8_t*>(dm);
      }
      // dict_strings becomes: base..., "" (NULL placeholder), extras...
      if (!extra.empty()) {
        c.dict_strings.resize(base_n);
        c.dict_strings.push_back(std::string());
        for (auto& e : extra) c.dict_strings.push_back(e);
      }
    }
    for (int depth = 0; depth < 2; depth++) {
      if (!c.delta[depth].present) continue;
      std::vector<DevDelta> one(1, c.delta[depth].dev);
      const DevDelta* dd = nullptr;
      rc = upload_vec(s, one, 16, &dd);
      if (rc) return rc;
      c.dev_delta[depth] = const_cast<DevDelta*>(dd);
    }
    c.dev.delta0 = c.dev_delta[0];
    c.dev.delta1 = c.dev_delta[1];
  }
  if (b->delete_buf) {   // [0][numBaseRows][numDeletes][positions]; the decoder walks to the buffer end
    const uint8_t* db = reinterpret_cast<const uint8_t*>(b->delete_buf);
    int64_t dlen = b->delete_len;
    std::vector<uint8_t> plain;
    if (dlen >= 8 && rd_i32(db) < 0) {   // stored compressed
      int rc0 = decompress_envelope_host(db, dlen, plain);
      if (rc0) return rc0;
      db = plain.data(); dlen = (int64_t)plain.size();
    }
    if (dlen < 12) return set_error(SD_ERR_INVALID, "delete buffer too short");
    const int n = (int)((dlen - 12) / 4);
    {   // ascending ordinals below num_rows (the kernels index tile bitmaps with them)
      int32_t prev = -1;
      for (int k = 0; k < n; k++) {
        const int32_t pos = rd_i32(db + 12 + 4 * (int64_t)k);
        if (pos <= prev || pos >= b->num_rows) return set_error(SD_ERR_INVALID, "delete positions must be ascending ordinals below %d (entry %d is %d)", b->num_rows, k, pos);
        prev = pos;
      }
    }
    uint8_t* p = nullptr;
    int rc = upload_bytes(s, db + 12, 4 * (size_t)n, 16, 0, &p);
    if (rc) return rc;
    sb->dev_deletes = reinterpret_cast<int32_t*>(p);
    sb->num_deletes = n;
  }
  if (b->stats_row && b->stats_len > 0) {
    sb->stats.assign(reinterpret_cast<const uint8_t*>(b->stats_row), reinterpret_cast<const uint8_t*>(b->stats_row) + b->stats_len);
    sb->stats_ncols = b->stats_ncols;
  }
  s->span_h0 = nullptr;
  // ownership rule: the caller's buffers may be released when this call returns (unless it retains them)
  if (!s->retain_buffers) {
    SD_CUDA(cudaStreamSynchronize(s->copy_stream));
    for (int k = 0; k + 1 < s->num_copy_streams; k++) SD_CUDA(cudaStreamSynchronize(s->extra_streams[k]));
    // scan images of a put whose bytes are all on the device now (one with LZ4 payloads still to expand keeps the verbatim
    // path, as does an asynchronous put of retained buffers)
    if (images && s->pending_lz4.size() == lz4_before) {
      int rc = build_images(s, s->copy_stream, {sb.get()}, true);
      if (rc) return rc;
    }
  }
  s->batches.push_back(std::move(sb));
  s->version++;
  return 0;
}

}  // namespace sd

// ---- C ABI: store ------------------------------------------------------------------------------------
extern "C" {

const char* sd_last_error(void) { return sd::last_error_cstr(); }

int sd_host_alloc(int64_t bytes, void** out) {
  if (!out || bytes < 0) return sd::set_error(SD_ERR_INVALID, "sd_host_alloc: bad arguments");
  SD_CUDA(cudaHostAlloc(out, (size_t)(bytes > 0 ? bytes : 1), cudaHostAllocDefault));
  return 0;
}
void sd_host_free(void* p) { if (p) cudaFreeHost(p); }
int sd_host_register(void* p, int64_t bytes) {
  if (!p || bytes <= 0) return sd::set_error(SD_ERR_INVALID, "sd_host_register: bad arguments");
  SD_CUDA(cudaHostRegister(p, (size_t)bytes, cudaHostRegisterDefault));
  return 0;
}
int sd_host_unregister(void* p) {
  if (!p) return sd::set_error(SD_ERR_INVALID, "sd_host_unregister: null");
  SD_CUDA(cudaHostUnregister(p));
  return 0;
}

int sd_store_create(int device, int32_t ncols, const sd_column* schema, sd_store** out) {
  if (!out || ncols < 0 || (ncols > 0 && !schema)) return sd::set_error(SD_ERR_INVALID, "sd_store_create: bad arguments");
  for (int32_t c = 0; c < ncols; c++)
    if (schema[c].type == SD_DECIMAL && (schema[c].precision < 0 || schema[c].precision > 38))
      return sd::set_error(SD_ERR_INVALID, "sd_store_create: DECIMAL column %d needs precision <= 38 (got %d)", c, schema[c].precision);
  int ndev = 0;
  SD_CUDA(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) return sd::set_error(SD_ERR_INVALID, "sd_store_create: device %d of %d", device, ndev);
  SD_CUDA(cudaSetDevice(device));
  sd_store* s = new sd_store();
  s->device = device;
  s->arena.device = device;
  s->arena.compressible = true;
  if (const char* env = getenv("SD_TUNE_STORE_SLAB_MB")) {   // (tests: stores of many small slabs)
    const long v = atol(env);
    if (v >= 2 && v <= 4096) s->arena.slab_bytes = size_t(v) << 20;
  }
  s->lz4_stage.device = device;
  s->lz4_stage.slab_bytes = size_t(256) << 20;
  s->schema.assign(schema, schema + ncols);
  cudaError_t e = cudaStreamCreateWithFlags(&s->copy_stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) { delete s; return sd::set_error(SD_ERR_CUDA, "cudaStreamCreate failed: %s", cudaGetErrorString(e)); }
  if (const char* env = getenv("SD_TUNE_COPY_STREAMS")) {
    const int v = atoi(env);
    if (v >= 2 && v <= 5) {
      s->num_copy_streams = v;
      for (int k = 0; k + 1 < v; k++) { cudaStreamCreateWithFlags(&s->extra_streams[k], cudaStreamNonBlocking); cudaEventCreateWithFlags(&s->extra_done[k], cudaEventDisableTiming); }
    }
  }
  *out = s;
  return 0;
}

int sd_store_put_batch(sd_store* s, const sd_batch* b) {
  if (!s || !b) return sd::set_error(SD_ERR_INVALID, "sd_store_put_batch: null argument");
  if (b->ncols != (int)s->schema.size()) return sd::set_error(SD_ERR_INVALID, "sd_store_put_batch: batch has %d columns, table schema %zu", b->ncols, s->schema.size());
  return sd::store_put(s, b, nullptr, true);
}

int sd_store_num_batches(sd_store* s, int64_t* out) { std::lock_guard<std::mutex> lock(s->mu); *out = (int64_t)s->batches.size(); return 0; }
int sd_store_bytes(sd_store* s, int64_t* out) { std::lock_guard<std::mutex> lock(s->mu); *out = (int64_t)s->arena.used; return 0; }
int sdx_store_memory_info(sd_store* s, int64_t* compressible_bytes, int64_t* slab_bytes) {
  if (!s || !compressible_bytes || !slab_bytes) return sd::set_error(SD_ERR_INVALID, "sdx_store_memory_info: null argument");
  std::lock_guard<std::mutex> lock(s->mu);
  *compressible_bytes = 0;
  *slab_bytes = 0;
  for (const auto& sl : s->arena.slabs) {
    *slab_bytes += (int64_t)sl.bytes;
    if (sl.compressed) *compressible_bytes += (int64_t)sl.bytes;
  }
  return 0;
}

void sd_store_destroy(sd_store* s) {
  if (!s) return;
  cudaSetDevice(s->device);
  if (s->copy_stream) cudaStreamDestroy(s->copy_stream);
  if (s->d_lz4_error) cudaFree(s->d_lz4_error);
  if (s->lz4_copied) cudaEventDestroy(s->lz4_copied);
  for (int k = 0; k < sd_store::LZ4_STREAMS; k++) {
    if (s->lz4_streams[k]) { cudaStreamSynchronize(s->lz4_streams[k]); cudaStreamDestroy(s->lz4_streams[k]); }
    if (s->lz4_done[k]) cudaEventDestroy(s->lz4_done[k]);
  }
  if (s->copies_done) cudaEventDestroy(s->copies_done);
  if (s->enc_stream) cudaStreamDestroy(s->enc_stream);
  if (s->enc_event) cudaEventDestroy(s->enc_event);
  delete s;
}

int sdx_store_batch_info(sd_store* s, int64_t batch_index, int32_t* num_rows, int32_t* bucket_id, int64_t* batch_id) {
  if (!s) return sd::set_error(SD_ERR_INVALID, "null store");
  std::lock_guard<std::mutex> lock(s->mu);
  if (batch_index < 0 || batch_index >= (int64_t)s->batches.size()) return sd::set_error(SD_ERR_INVALID, "batch index out of range");
  const sd::StoredBatch& b = *s->batches[batch_index];
  if (num_rows) *num_rows = b.num_rows;
  if (bucket_id) *bucket_id = b.bucket_id;
  if (batch_id) *batch_id = b.batch_id;
  return 0;
}

int sdx_store_get_buffer(sd_store* s, int64_t batch_index, int32_t table_col, void* out, int64_t cap, int64_t* out_len) {
  if (!s) return sd::set_error(SD_ERR_INVALID, "null store");
  std::lock_guard<std::mutex> lock(s->mu);
  if (batch_index < 0 || batch_index >= (int64_t)s->batches.size()) return sd::set_error(SD_ERR_INVALID, "batch index out of range");
  const sd::StoredBatch& b = *s->batches[batch_index];
  if (table_col < 0 || table_col >= (int)b.cols.size() || !b.cols[table_col].present || !b.cols[table_col].dev_base)
    return sd::set_error(SD_ERR_INVALID, "column %d not resident", table_col);
  const sd::StoredCol& c = b.cols[table_col];
  { int rc = sd::store_flush_lz4(s); if (rc) return rc; rc = sd::store_lz4_check(s); if (rc) return rc; }
  *out_len = c.len;
  if (cap < c.len) return sd::set_error(SD_ERR_OVERFLOW, "buffer too small");
  SD_CUDA(cudaSetDevice(s->device));
  SD_CUDA(cudaMemcpy(out, c.dev_base, (size_t)c.len, cudaMemcpyDeviceToHost));
  return 0;
}

}  // extern "C"
