// sd_host.h -- internal host-side declarations shared by the engine translation units.
#ifndef SD_HOST_H
#define SD_HOST_H

#include <cuda_runtime.h>

#include <atomic>
#include <climits>
#include <cstdint>
#include <functional>
#include <memory>
#include <mutex>
#include <set>
#include <string>
#include <type_traits>
#include <unordered_map>
#include <vector>

#include "../../include/snappy_gpu.h"
#include "sd_codegen.h"
#include "sd_device.h"

namespace sd {

// ---- errors -------------------------------------------------------------------------------------
int set_error(int code, const char* fmt, ...);
#define SD_CUDA(call)                                                                         \
  do {                                                                                        \
    cudaError_t e__ = (call);                                                                 \
    if (e__ != cudaSuccess)                                                                   \
      return sd::set_error(SD_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

// ---- kernel registry ------------------------------------------------------------------------------
struct KernelEntry {
  std::string signature;
  const void* func;      // &scan_aggregate_kernel<PLAN> (runtime API launch)
  void* drv_func;        // CUfunction for NVRTC-compiled plans
  size_t tile_smem;      // sizeof(TileSmem<PLAN>) rounded up to 16
  int staged = 0;        // PLAN::STAGES > 0: producer warp + shared-memory ring (block = THREADS + 32)
  size_t stage_bytes = 0;
  int tile_rows = 0;     // THREADS * PLAN::RPT (set by the engine when it resolves the kernel)
  // a dense group-by's staged-only variant: its kernel for two CTAs per SM (scan_aggregate_kernel_2cta), else null
  const void* func2 = nullptr;
  void* drv_func2 = nullptr;
  std::string origin;    // "aot" | "jit"
  std::string name;      // Plan_<fnv1a(signature)>: the generated struct's name
};
std::vector<KernelEntry>& kernel_registry();
std::string plan_struct_name(const std::string& signature);
struct AotRegistrar {
  AotRegistrar(const char* signature, const void* func, size_t tile_smem, int staged, size_t stage_bytes, const void* func2);
};
// set the dynamic shared-memory limit and query CTAs/SM; launch (runtime API for AOT, driver API for JIT)
// two_cta: the entry's two-CTA kernel (func2 / drv_func2) instead of its kernel
int kernel_prepare(const KernelEntry& k, bool two_cta, size_t smem, int* ctas_per_sm);
int kernel_local_bytes(const KernelEntry& k, bool two_cta, size_t* bytes);   // local memory per thread (spills, stack)
inline int kernel_block_threads(const KernelEntry& k) { return THREADS + (k.staged ? 32 : 0); }
int kernel_launch(const KernelEntry& k, bool two_cta, int grid, size_t smem, cudaStream_t stream, void** args);
// NVRTC path (sd_jit.cpp): compile `spec.source` against the embedded kernel headers.
int jit_compile(const PlanSpec& spec, int device, KernelEntry& out);

// ---- MODE_HASH group table housekeeping (sd_hash.cu) ------------------------------------------------
// nshift: K words per entry of moment aggregates (t.shifts; sd_device.h SHIFT_EMPTY), copied out to out_shifts by the compaction
int hash_table_init(cudaStream_t stream, const HashTable& t, uint32_t capacity, int nslot, const uint64_t* d_ident, int nshift);
int hash_table_compact(cudaStream_t stream, const HashTable& t, uint32_t capacity, int nk, int nslot, int64_t* out_keys,
                       uint32_t* out_knull, uint64_t* out_vals, uint32_t* d_cursor, int nshift, uint64_t* out_shifts);
// ---- grouping-sets roll-up (sd_rollup.cu): fine groups of the plain GROUP BY scan -> a hash table keyed by (keys, gid) ---------
struct RollupArgs {
  // fine groups: compacted hash entries (keys != nullptr: keys [nfine][nk], knull) or the dense [nfine][ns] table (keys == nullptr:
  // entry e is the mixed-radix index over radix[], dictionary id null_id[k] is key k's NULL)
  const int64_t* keys;
  const uint32_t* knull;
  const uint64_t* vals;          // [nfine][ns]
  const uint64_t* shifts;        // [nfine][nsh] K words
  int32_t radix[MAX_KEYS];
  int32_t null_id[MAX_KEYS];
  uint32_t nfine;
  int32_t nk, ns, nsh;
  int32_t rows_slot;             // an entry whose row count is 0 does not exist
  uint32_t strmask;              // keys held by reference (compared by their bytes)
  const uint32_t* masks;         // [nsets]
  int32_t nsets;
  const int32_t* slot_op;        // [ns] SLOT_*
  const int32_t* slot_role;      // [ns] -1 plain; (shift << 3) | j: S_j of a shift; -2 - q: S_xy of pair q
  const int32_t* shift_count;    // [nsh] the slot holding n of the shift's input
  const int32_t* shift_pow;      // [nsh][4] S_1..S_4 slots
  const int32_t* pair_x;         // [npair] shift of x
  const int32_t* pair_y;         // [npair] shift of y
  HashTable out;                 // nk + 1 keys (the last is gid), ns slots, nsh K words per entry
};
int rollup_launch(cudaStream_t stream, const RollupArgs& a);

// strings held by reference -> host: d_recs[i * stride] = device address of a [len:int32][bytes] record (0: none)
int fetch_string_records(cudaStream_t stream, const int64_t* d_recs, int64_t n, int64_t stride, std::vector<std::string>& out);

// ---- sd_rows.cu: projection records -> UnsafeRows on the device -------------------------------------------------------------
constexpr int ROW_MAX_FIELDS = 32;   // one lane per field; the record's null bits are 32 wide
enum { ROW_KIND_8 = 0, ROW_KIND_BOOL = 1, ROW_KIND_1 = 2, ROW_KIND_2 = 3, ROW_KIND_4 = 4, ROW_KIND_FLOAT = 5, ROW_KIND_STRING = 6 };
// where the strings of one projected STRING column of one batch live on the device
struct RowStrSrc {
  const uint8_t* base;        // dictionary: the column's uploaded buffer; raw strings: its [len][bytes] body
  const int32_t* rec_off;     // dictionary: offset of each code's [len][bytes] record from base; nullptr: raw (the value IS the offset)
  int32_t null_code;          // dictionary code that stands for NULL (-1: none)
  int32_t n;                  // dictionary entries
};
struct RowWriterBuffers {
  int64_t* d_offs = nullptr; size_t offs_cap = 0;
  void* d_tmp = nullptr; size_t tmp_cap = 0;
  uint8_t* d_rows = nullptr; size_t rows_cap = 0;
  int32_t* d_err = nullptr;
  RowStrSrc* d_src = nullptr; size_t src_cap = 0;       // [batches of the execution][string fields]
  int32_t* d_recoff = nullptr; size_t recoff_cap = 0;   // the rec_off tables, back to back
  std::vector<const void*> src_key;                       // the batches d_src / d_recoff were built for
  void release();
};
int device_write_rows(cudaStream_t st, const uint64_t* d_recs, int64_t count, int np, const uint8_t* kinds, int nbatches,
                      RowWriterBuffers& b, int64_t* total_out);

// ---- on-device LZ4 (sd_lz4.cu) ---------------------------------------------------------------------------
struct Lz4Job { const uint8_t* src; uint8_t* dst; int64_t src_len; int64_t dst_len; };
int64_t lz4_decode_prefix(const uint8_t* src, int64_t src_len, uint8_t* dst, int64_t want);
// host Snappy (raw format) decoder: returns the uncompressed length or -1 (sd_lz4.cu)
int64_t snappy_decode(const uint8_t* src, int64_t src_len, uint8_t* dst, int64_t dst_cap);
// a stored buffer [-codecId][uncompressedLen][payload] (CompressionUtils.scala:53-61) -> its uncompressed bytes, on the host
int decompress_envelope_host(const uint8_t* buf, int64_t len, std::vector<uint8_t>& out);
int lz4_launch(cudaStream_t stream, const Lz4Job* d_jobs, int njobs, unsigned int* d_error);

// ---- NCCL behind sd_comm (sd_nccl.cpp; dlopen'ed) --------------------------------------------------------
int comm_unique_id(void* out128);
int comm_init(const void* id128, int rank, int world, void** out);
void comm_destroy(void* c);
int comm_all_gather_bytes(void* c, const void* d_send, void* d_recv, size_t bytes_per_rank, cudaStream_t stream);

// ---- device memory arena: bump allocation out of large slabs ---------------------------------------
// one allocation of a store's arena that a batch version owns (sd_reclaim.cu moves and frees by these)
struct Extent { uint8_t* ptr; size_t bytes; };
struct Arena {
  int device = 0;
  size_t slab_bytes = size_t(512) << 20;
  // slabs from cuMemCreate with generic compression requested, where the device reports support for it: the hardware
  // compresses them between L2 and DRAM, so a scan of compressible bytes moves fewer DRAM bytes; what kernels and copies
  // see is unchanged.  Set for the resident store only; everything else stays on cudaMalloc.
  bool compressible = false;
  struct Slab {
    uint8_t* base;
    size_t bytes;
    bool vmm;                   // cuMemCreate + cuMemMap (else cudaMalloc)
    bool compressed;            // the driver granted generic compression
    unsigned long long handle;  // CUmemGenericAllocationHandle of a vmm slab
    size_t used;                // bytes allocated out of it
  };
  std::vector<Slab> slabs;
  size_t cur_slab = 0;
  size_t cur_off = 0;
  size_t used = 0;
  // non-null: every allocation is appended here as an extent (ExtentRecorder scopes it to one batch version)
  std::vector<Extent>* record = nullptr;
  // returns p with (p + misalign) % align == 0, or nullptr (error set)
  uint8_t* alloc(size_t n, size_t align = 256, size_t misalign = 0);
  void reset();     // keep slabs, forget allocations
  void release();   // free slabs
  // stop allocating from the current slab: the next allocation opens a fresh one
  void close_slab() { cur_slab = slabs.size(); cur_off = 0; }
  // take slab i out of the arena (its allocated bytes leave `used`); the caller frees it with free_slab
  Slab detach_slab(size_t i);
  static void free_slab(int device, const Slab& s);
  ~Arena() { release(); }
};
struct ExtentRecorder {
  Arena& a;
  ExtentRecorder(Arena& arena, std::vector<Extent>* to) : a(arena) { a.record = to; }
  ~ExtentRecorder() { a.record = nullptr; }
};

// page-locked host staging for small uploads (descriptors, tables) that must not block the submitting thread:
// copies from it are truly asynchronous, and the memory stays valid until reset()
struct PinnedArena {
  size_t slab_bytes = size_t(4) << 20;
  std::vector<std::pair<uint8_t*, size_t>> slabs;
  size_t cur_slab = 0, cur_off = 0;
  uint8_t* alloc(size_t n);   // 16-byte aligned, nullptr on failure (error set)
  void reset() { cur_slab = 0; cur_off = 0; }
  ~PinnedArena();
};

// ---- resident batches ------------------------------------------------------------------------------
struct StoredDelta {
  bool present = false;
  DevDelta dev;                           // device pointers
  int64_t len = 0;
  int32_t nbase = 0;                      // numBaseRows of the header
  int64_t body_off = 0;                   // offset of the values (dictionary) in the reference layout
  std::vector<std::string> dict_strings;  // STRING values dictionary
};

struct StoredCol {
  bool present = false;
  std::string unsupported;                // non-empty: reason the GPU path cannot scan this column
  int64_t len = 0;
  int64_t algo_bytes = 0;                 // len - 8 - dictionary bytes (SURVEY.md 8d)
  uint8_t* dev_base = nullptr;            // device copy of the whole buffer
  int64_t body_off = 0;                   // offset of the first value / index
  DevCol dev;                             // device view (delta pointers filled per plan)
  std::vector<std::string> dict_strings;  // STRING dictionary (or distinct RLE run strings)
  std::vector<int64_t> dict_rec_off;      // per dict_strings entry: offset of its [len][bytes] record in the buffer (-1: none)
  std::vector<int64_t> dict_rec_ptr;      // per unified code: device address of the record (0: NULL placeholder) -- string keys by reference
  bool raw_str = false;                   // Uncompressed variable-width STRING body (dev.enc == ENC_STR_RAW)
  bool has_nulls = false;
  StoredDelta delta[2];
  DevDelta* dev_delta[2] = {nullptr, nullptr};   // DevDelta structs resident on the device
  bool fast = false;                      // vector fast path applies
  // scan image (sd_image.cu; DevCol.img): element bytes of the verbatim values it reproduces, whether it is a dictionary of
  // bit patterns (else a frame of reference), and the arena bytes it takes
  int32_t img_ew = 0;
  bool img_dict = false;
  int64_t img_bytes = 0;
};

inline uint64_t next_batch_uid() { static std::atomic<uint64_t> n{1}; return n.fetch_add(1, std::memory_order_relaxed); }
struct StoredBatch {
  uint64_t uid = next_batch_uid();        // never reused (an address can be): key of per-plan caches built from a batch
  int32_t num_rows = 0;
  int32_t bucket_id = 0;
  int64_t batch_id = 0;
  std::vector<StoredCol> cols;            // by table column
  std::vector<uint8_t> stats;             // stats UnsafeRow (host copy)
  int32_t stats_ncols = 0;
  int32_t* dev_deletes = nullptr;
  int32_t num_deletes = 0;
  bool has_deltas = false;
  bool positional = false;                // cols are indexed by the plan's scan column (private store)
  bool gone = false;                      // every row deleted (ColumnDelta.checkBatchDeleted): no scan reads it
  // the arena allocations this version's device pointers lie in (a new version inherits those of the columns it keeps;
  // store_install drops the ones no pointer refers to any more)
  std::vector<Extent> extents;
  int64_t retired_at = -1;                // store version that replaced or removed it (scans of an older snapshot may read it)
};

// Every device pointer a batch version owns, in one place: the reclaim's inventory and its rebase both walk this list
// (sd_reclaim.cu).  f(uintptr_t address, int table_col, const char* field) returns the address the field is to hold; the
// batch's delete mask reports column -1.  The device-resident DevDelta structs (dev_delta[]) hold copies of the host
// StoredDelta::dev pointers; whoever moves them rewrites them from the host copies.
template <class F>
void visit_device_pointers(StoredBatch& b, F&& f) {
  auto one = [&](auto& field, int col, const char* what) {
    if (!field) return;
    typedef typename std::remove_reference<decltype(field)>::type P;
    field = (P)f((uintptr_t)field, col, what);
  };
  for (int c = 0; c < (int)b.cols.size(); c++) {
    StoredCol& sc = b.cols[c];
    if (!sc.present) continue;
    one(sc.dev_base, c, "dev_base");
    one(sc.dev.data, c, "data");
    one(sc.dev.nulls, c, "nulls");
    one(sc.dev.tile_nulls, c, "tile_nulls");
    one(sc.dev.dict, c, "dict");
    one(sc.dev.run_ends, c, "run_ends");
    one(sc.dev.delta0, c, "delta0");
    one(sc.dev.delta1, c, "delta1");
    one(sc.dev.img, c, "img");
    one(sc.dev.img_tab, c, "img_tab");
    for (int d = 0; d < 2; d++) {
      StoredDelta& sd = sc.delta[d];
      if (sd.present) {
        one(sd.dev.positions, c, "delta positions");
        one(sd.dev.data, c, "delta data");
        one(sd.dev.nulls, c, "delta nulls");
        one(sd.dev.dict, c, "delta dict");
      }
      one(sc.dev_delta[d], c, "dev_delta");
    }
    for (int64_t& r : sc.dict_rec_ptr) one(r, c, "dict_rec_ptr");
  }
  one(b.dev_deletes, -1, "dev_deletes");
}
// Scan images of the given fresh batch versions (sd_image.cu): every NOT NULL column without NULLs in the batch whose values
// fit a narrower byte-aligned form gets one, built and verified on the device, placed in the store's arena as extents of its
// version.  Columns that already have an image keep it.  The batches' bytes are complete in stream order on `st`; the
// batches are not yet visible to scans.  `locked`: the caller holds s->mu (else it is taken for the arena placement only,
// so that scans are not held up by the build).  Synchronises `st`.
int build_images(sd_store* s, cudaStream_t st, const std::vector<StoredBatch*>& batches, bool locked);
// image choice for a column's values: width in bytes (0: none) of a dictionary image (float kinds, `ndistinct` distinct bit
// patterns) or a frame of reference over [lo, hi] (integral kinds, element width ew)
int image_width(bool dict, int ew, uint64_t ndistinct, int64_t lo, int64_t hi);
// drop the extents no device pointer of the version lies in (those a replaced delta / mask / column left behind)
void prune_extents(StoredBatch& b);

// Scans that may still read a store's memory: the store version each one saw when it took its snapshot.  Shared between
// the store and the plans that scanned it (either may be destroyed first).
struct ScanPins {
  std::mutex mu;
  std::multiset<int64_t> versions;
  int64_t oldest() {
    std::lock_guard<std::mutex> lock(mu);
    return versions.empty() ? INT64_MAX : *versions.begin();
  }
};
// the pins a plan holds: at most one per store, the oldest (taken at its first snapshot of the execution)
struct HeldPins {
  std::vector<std::pair<std::shared_ptr<ScanPins>, int64_t>> held;
  void take(const std::shared_ptr<ScanPins>& r, int64_t version) {
    for (auto& h : held) if (h.first == r) return;
    std::lock_guard<std::mutex> lock(r->mu);
    r->versions.insert(version);
    held.emplace_back(r, version);
  }
  void release() {
    for (auto& h : held) {
      std::lock_guard<std::mutex> lock(h.first->mu);
      auto it = h.first->versions.find(h.second);
      if (it != h.first->versions.end()) h.first->versions.erase(it);
    }
    held.clear();
  }
  ~HeldPins() { release(); }
};

}  // namespace sd

struct sd_store {
  // ingest (sd_store_put_batch) may run concurrently with scans: `mu` guards batches / arena / version / the LZ4 queues.  A scan
  // works on the SNAPSHOT of batch pointers it takes under the lock when it starts (a batch becomes visible only after its
  // bytes have reached the device; a batch replaced or removed by UPDATE / DELETE / compaction stays alive in `retired`).
  std::mutex mu;
  int device = 0;
  std::vector<sd_column> schema;
  sd::Arena arena;
  cudaStream_t copy_stream = nullptr;
  // extra H2D streams (SD_TUNE_COPY_STREAMS > 1): large buffer copies rotate over them
  cudaStream_t extra_streams[4] = {nullptr, nullptr, nullptr, nullptr};
  int num_copy_streams = 1;
  int next_stream = 0;
  cudaEvent_t extra_done[4] = {nullptr, nullptr, nullptr, nullptr};
  std::vector<std::unique_ptr<sd::StoredBatch>> batches;
  // UPDATE / DELETE / compaction / reclaim replace a batch by a new version at the same index (compaction also drops fully
  // deleted batches); the old one stays alive here (scans hold raw pointers into their snapshot) until sd_store_reclaim finds
  // that no open scan can read it, or the store is destroyed.  `mutate_mu` serialises the statements, compactions and
  // reclaims on this store.
  std::vector<std::unique_ptr<sd::StoredBatch>> retired;
  std::mutex mutate_mu;
  // the open scans of this store (taken with the snapshot under `mu`, released when the scan's result is materialised)
  std::shared_ptr<sd::ScanPins> pins = std::make_shared<sd::ScanPins>();
  int64_t version = 0;
  int64_t h2d_bytes = 0;
  bool retain_buffers = false;   // SD_OPT_RETAIN_BUFFERS: no per-put synchronisation of the copy stream
  cudaEvent_t copies_done = nullptr;
  // compressed payloads waiting to be expanded on the device (one launch for many buffers)
  std::vector<sd::Lz4Job> pending_lz4;
  sd::Arena lz4_stage;
  unsigned int* d_lz4_error = nullptr;
  int64_t lz4_buffers = 0, lz4_in_bytes = 0, lz4_out_bytes = 0;
  // expansions are queued on a few streams of their own so that the launches of successive flushes (each one as
  // long as its longest buffer) overlap each other and the copies that follow
  static constexpr int LZ4_STREAMS = 12;   // enough launches in flight to keep ~2800 buffers resident with 256 MB flushes
  cudaStream_t lz4_streams[LZ4_STREAMS] = {};
  cudaEvent_t lz4_done[LZ4_STREAMS] = {};
  bool lz4_used[LZ4_STREAMS] = {};
  cudaEvent_t lz4_copied = nullptr;
  int lz4_next = 0;
  // compressed payloads of one batch that lie (almost) back to back in host memory travel as ONE copy
  const uint8_t* span_h0 = nullptr; uint8_t* span_d0 = nullptr; size_t span_len = 0;
  sd::PinnedArena lz4_jobs_host;
  sd::PinnedArena enc_host;        // sd_encode.cu: prefixes / descriptors on their way to the device
  std::mutex enc_mu;               // one encoder at a time per store; `mu` is taken only to lay the buffers out and to publish
  cudaStream_t enc_stream = nullptr;
  cudaEvent_t enc_event = nullptr;   // page-locked copies of the job lists (a pageable source would stall the caller per flush)
  // scan images (sd_image.cu): (batch, column) images whose device verification failed (the column keeps its verbatim path),
  // and the time spent building images
  int64_t image_mismatches = 0;
  double image_ms = 0;
};

namespace sd {
// upload one batch (columns by table ordinal of `schema`) into the store's arena; `images`: build its scan images (resident
// stores; the private store of sd_batch_submit scans each batch once and skips them)
int store_put(sd_store* s, const sd_batch* b, const int32_t* table_ordinals /* nullptr: identity */, bool images = false);
// queue the expansion of every pending compressed buffer (asynchronous; no-op when nothing is pending)
int store_flush_lz4(sd_store* s);
// make `stream` wait for every expansion queued so far
int store_lz4_order(sd_store* s, cudaStream_t stream);
// block until the queued expansions are done, release their staging memory, report a corrupt payload
int store_lz4_check(sd_store* s);

// records of an UPDATE / DELETE scan, on the device (sd_engine.cu; merged by sd_mutate.cu): `count` records of `rec_words`
// uint64 words, [batch << 32 | row][null bits][SET values]; the batch ordinal indexes `batches`
struct MutationScan {
  const uint64_t* records = nullptr;
  int64_t count = 0;
  int rec_words = 0;
  std::vector<const StoredBatch*> batches;
  cudaStream_t stream = nullptr;
  float scan_ms = 0;
};
int mutation_scan(sd_plan* p, sd_store* s, const int32_t* bucket_ids, int32_t nbuckets, const sd_literal* lits, int32_t nlits,
                  MutationScan* out);
// the analysed plan of a handle (sd_engine.cu)
const PlanSpec& plan_spec(const sd_plan* p);

// device scratch of one statement / compaction round, stream-ordered (cudaMallocAsync / cudaFreeAsync: no device-wide
// synchronisation, so queries running on other streams are not stalled by its allocations), released when it ends
struct DevScratch {
  cudaStream_t st = nullptr;
  std::vector<void*> ptrs;
  template <class T> int get(T** out, size_t bytes) {
    void* p = nullptr;
    SD_CUDA(cudaMallocAsync(&p, bytes ? bytes : 16, st));
    ptrs.push_back(p);
    *out = reinterpret_cast<T*>(p);
    return 0;
  }
  ~DevScratch() { for (void* p : ptrs) cudaFreeAsync(p, st); }
};

// install new batch versions and drop batches, all under ONE hold of the store's lock (a scan's snapshot sees every change
// or none): fresh[i].second replaces fresh[i].first at its index, `remove` leaves the store; the replaced and removed
// versions move to `retired` (scans of an older snapshot may still read them) marked with the new store version; the
// fresh versions' extents are pruned.  SD_ERR_STATE, nothing changed, when one of the named batches is no longer in the
// store (sd_store.cu)
typedef std::vector<std::pair<const StoredBatch*, std::unique_ptr<StoredBatch>>> FreshBatches;
int store_install(sd_store* s, FreshBatches& fresh, const std::vector<const StoredBatch*>& remove, const char* what);

// ---- the device encoder (sd_encode.cu): raw column values resident on the device -> encoded buffers in the store ---------
// Shared by ingest (sd_store_encode_batch, one batch) and compaction (sd_compact.cu, the columns of many batches at once).
// Per column: enc_null_words_many (null words + null count, one launch for all), read back fb / words (enc_queue_words), enc_layout under the store's lock (header,
// trimmed null words, dictionary in first-seen order; arena placement through store_register_encoded), then ONE
// enc_write launch for every column of the call (compacted values / bit set / dictionary indexes, min / max).
struct ColStat { bool present = false, has = false; int type = 0; uint64_t lo = 0, hi = 0; std::string slo, shi; int32_t nulls = 0; };
// stats UnsafeRow [count:int][(lower, upper, nullCount:int) per table column] (enc/ColumnEncoding.scala:1015-1036)
std::vector<uint8_t> stats_row_bytes(int32_t count, const std::vector<ColStat>& st);
// a stats row of ncols columns with a new count and the given columns' entries replaced; every other entry keeps its bytes
// (replaced STRING bounds are appended to the variable-length region)
void stats_row_replace(std::vector<uint8_t>& row, int ncols, int32_t count, const std::vector<std::pair<int, const ColStat*>>& entries);
struct EncJob {
  int table_col = 0, type = 0, n = 0;
  bool nullable = false;
  const uint8_t* d_values = nullptr;   // n values of the type's width (BOOLEAN: one byte); STRING: int32 "slot" per row
  const uint8_t* d_nulls = nullptr;    // n null flags (one byte, non-zero = NULL) or nullptr
  int32_t* d_slot_code = nullptr;      // STRING: slot -> dictionary index, filled by enc_layout from slot_codes
  int2* d_slot_pairs = nullptr;        // STRING: device room for slot_codes
  std::vector<std::string> dict;       // STRING: the distinct values in first-seen order
  std::vector<int2> slot_codes;        // STRING: (slot, dictionary index) of every distinct value
  // set by the encoder
  uint64_t* d_words = nullptr;         // null words (room for ceil(n / 64))
  int* d_fb = nullptr;                 // [0] nulls [1] last non-zero null word + 1 (zeroed by the caller)
  uint64_t* d_stat = nullptr;          // [0] lower [1] upper [2] non-null count
  int fb[2] = {0, 0};
  std::vector<uint64_t> words;         // the trimmed null words, read back
  uint8_t* d_body = nullptr;           // where enc_write puts the body
  int64_t body_len = 0;
};
typedef uint8_t* (*DevAllocFn)(void* ctx, size_t bytes);   // 16-byte aligned device scratch, nullptr on failure (error set)
// the null words of every job with nulls, in one launch (d_words / d_fb must be set, d_fb zeroed)
int enc_null_words_many(cudaStream_t st, const std::vector<EncJob*>& jobs, DevAllocFn alloc, void* ctx, PinnedArena& pin);
// after fb has been read back: queue the read-back of the trimmed null words of the jobs that hold NULLs (true: some were
// queued; the caller synchronises); *rc: error
bool enc_queue_words(cudaStream_t st, const std::vector<EncJob*>& jobs, int* rc);
// STRING: the dictionary in first-seen order from (slot, first position) of every distinct value -> j.dict, j.slot_codes
void enc_first_seen_dict(EncJob& j, std::vector<int2>& slot_first, const std::function<std::string(int slot, int first)>& value_of);
// lay one column out in the arena (caller holds s->mu): registers `sc`, queues the prefix upload, sets d_body and the stats
int enc_layout(sd_store* s, cudaStream_t st, PinnedArena& pin, EncJob& j, StoredCol& sc, ColStat& cs);
// write every job's body in one launch and finish the stats (the caller has ordered `st` after the side uploads)
// (ev_begin / ev_end, when given, are recorded around the launch)
int enc_write(cudaStream_t st, DevAllocFn alloc, void* ctx, PinnedArena& pin, const std::vector<EncJob*>& jobs,
              const std::vector<ColStat*>& stats, cudaEvent_t ev_begin = nullptr, cudaEvent_t ev_end = nullptr);
}

#endif
