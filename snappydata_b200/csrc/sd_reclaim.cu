// sd_reclaim.cu -- giving back the device memory of superseded batch versions (sd_store_reclaim).
//
// The store's arena is bump-allocated out of 512 MB slabs, and UPDATE / DELETE / compaction never write in place: every
// version they replace stays readable for the scans of older snapshots.  Reclaim frees what nobody can read any more:
//   1. inventory  the extents (arena allocations) of every current version, and of every retired version that an open
//                 scan may still read (ScanPins); retired versions no scan can read are destroyed.  Every device pointer a
//                 current version holds must lie in one of its own extents -- checked before anything is copied;
//   2. select     slabs without live bytes are freed at once; slabs whose live bytes are at most max_live_fraction of
//                 their size are evacuated, emptiest first, in rounds of at most one destination slab;
//   3. copy       one launch per round moves every extent of a current version that lies in the round's source slabs,
//                 plus the small DevDelta structs of the batches it touches (rewritten with rebased pointers).  A
//                 destination keeps its extent's address modulo 256, so every alignment the layout chose survives;
//   4. install    new versions of the round's batches (same bytes at new addresses, new uid) in one hold of the store's
//                 lock: a scan sees the whole round or none of it;
//   5. free       the source slabs no open scan can read; the others are deferred to a later call.
#include <algorithm>
#include <chrono>
#include <map>

#include "sd_host.h"

namespace sd {
const char* last_error_cstr();
namespace {

// ---- the copy kernel ----------------------------------------------------------------------------------------------------
// Chunks of CP_CHUNK bytes over the prefix sum of the extents' sizes; a CTA binary-searches the extent of each chunk it
// takes.  The 16-byte-aligned middle of a chunk goes global -> shared -> global through a ring of bulk copies (loads
// complete on an mbarrier, stores are bulk groups; a stage is refilled once its store has read it); the unaligned head and
// tail (< 16 bytes each) are plain byte copies.  Both ends are compressible slabs, where direct loads of incompressible
// bytes run well below the bulk path (DESIGN.md section 4).
constexpr int CP_THREADS = 32;
constexpr int CP_STAGES = 4;
constexpr int CP_STAGE_BYTES = 16 << 10;
constexpr int64_t CP_CHUNK = 256 << 10;

struct CopyJob { const uint8_t* src; uint8_t* dst; int64_t bytes; };

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred P1;\n\tLAB_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\tbra LAB_WAIT;\n\tDONE:\n\t}" ::"r"(bar), "r"(parity) : "memory");
}

__global__ void __launch_bounds__(CP_THREADS) reclaim_copy_kernel(const CopyJob* __restrict__ jobs, const int64_t* __restrict__ first_chunk,
                                                                  int njobs, int64_t nchunks) {
  extern __shared__ __align__(128) uint8_t ring[];   // CP_STAGES x CP_STAGE_BYTES
  __shared__ __align__(8) uint64_t bar[CP_STAGES];
  const int lane = threadIdx.x;
  if (lane == 0) {
    for (int s = 0; s < CP_STAGES; s++) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_addr(&bar[s])) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  uint32_t parity = 0;   // bit s: parity of stage s's next completion
  for (int64_t c = blockIdx.x; c < nchunks; c += gridDim.x) {
    int lo = 0, hi = njobs - 1;   // the last job whose first chunk is <= c
    while (lo < hi) {
      const int m = (lo + hi + 1) >> 1;
      if (first_chunk[m] <= c) lo = m; else hi = m - 1;
    }
    const CopyJob j = jobs[lo];
    const int64_t off = (c - first_chunk[lo]) * CP_CHUNK;
    const int64_t len = min(CP_CHUNK, j.bytes - off);
    const uint8_t* src = j.src + off;
    uint8_t* dst = j.dst + off;   // same address modulo 256 as src
    const uintptr_t s0 = (uintptr_t)src, s1 = s0 + (uintptr_t)len;
    uintptr_t a = (s0 + 15) & ~uintptr_t(15), b = s1 & ~uintptr_t(15);
    if (a >= b) a = b = s1;        // no aligned middle: all of it is head
    const int64_t head = (int64_t)(a - s0), mid = (int64_t)(b - a), tail = (int64_t)(s1 - b);
    for (int64_t i = lane; i < head; i += CP_THREADS) dst[i] = src[i];
    for (int64_t i = lane; i < tail; i += CP_THREADS) dst[head + mid + i] = src[head + mid + i];
    if (lane == 0 && mid > 0) {
      const int np = (int)((mid + CP_STAGE_BYTES - 1) / CP_STAGE_BYTES);
      auto piece = [&](int i) { return (uint32_t)min((int64_t)CP_STAGE_BYTES, mid - (int64_t)i * CP_STAGE_BYTES); };
      auto load = [&](int i) {
        const int s = i % CP_STAGES;
        const uint32_t n = piece(i), b_s = smem_addr(&bar[s]);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b_s), "r"(n) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(smem_addr(ring + s * CP_STAGE_BYTES)), "l"(src + head + (int64_t)i * CP_STAGE_BYTES), "r"(n), "r"(b_s)
                     : "memory");
      };
      for (int i = 0; i < np && i < CP_STAGES; i++) load(i);
      for (int i = 0; i < np; i++) {
        const int s = i % CP_STAGES;
        mbar_wait(smem_addr(&bar[s]), (parity >> s) & 1u);
        parity ^= 1u << s;
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                     ::"l"(dst + head + (int64_t)i * CP_STAGE_BYTES), "r"(smem_addr(ring + s * CP_STAGE_BYTES)), "r"(piece(i))
                     : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        if (i >= 1 && i - 1 + CP_STAGES < np) {
          asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");   // the store of piece i - 1 has read its stage
          load(i - 1 + CP_STAGES);
        }
      }
      asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // every stage is free for the next chunk
    }
    __syncwarp();
  }
  if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // the stores are done before the CTA leaves
}

constexpr size_t CP_SMEM = (size_t)CP_STAGES * CP_STAGE_BYTES;

// ---- host side ----------------------------------------------------------------------------------------------------------
struct Timing { double plan_ms = 0, copy_ms = 0, install_ms = 0, free_ms = 0, total_ms = 0, rounds = 0; };
thread_local Timing g_timing;

double ms_since(std::chrono::steady_clock::time_point t) {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t).count();
}

bool by_ptr(const Extent& a, const Extent& b) { return a.ptr < b.ptr; }

// the extent of `sorted` that holds address a, or nullptr
const Extent* containing(const std::vector<Extent>& sorted, uintptr_t a) {
  auto it = std::upper_bound(sorted.begin(), sorted.end(), a, [](uintptr_t x, const Extent& e) { return x < (uintptr_t)e.ptr; });
  if (it == sorted.begin()) return nullptr;
  --it;
  return a < (uintptr_t)it->ptr + it->bytes ? &*it : nullptr;
}

// the index of the slab holding address a (slabs sorted by base), or -1
int slab_of(const std::vector<Arena::Slab>& sorted, const uint8_t* a) {
  auto it = std::upper_bound(sorted.begin(), sorted.end(), a, [](const uint8_t* x, const Arena::Slab& s) { return x < s.base; });
  if (it == sorted.begin()) return -1;
  --it;
  return a < it->base + it->bytes ? (int)(it - sorted.begin()) : -1;
}

// destroy the retired versions no open scan can read (caller holds s->mu)
void drop_unreadable_retired(sd_store* s) {
  const int64_t oldest = s->pins->oldest();
  size_t k = 0;
  for (size_t i = 0; i < s->retired.size(); i++)
    if (s->retired[i]->retired_at > oldest) s->retired[k++] = std::move(s->retired[i]);
  s->retired.resize(k);
}

// every extent of the current versions and of the retired versions still kept, sorted, one entry per allocation
// (caller holds s->mu)
std::vector<Extent> live_extents(sd_store* s, bool with_retired) {
  std::vector<Extent> all;
  for (auto& b : s->batches) all.insert(all.end(), b->extents.begin(), b->extents.end());
  if (with_retired) for (auto& b : s->retired) all.insert(all.end(), b->extents.begin(), b->extents.end());
  std::sort(all.begin(), all.end(), by_ptr);
  all.erase(std::unique(all.begin(), all.end(), [](const Extent& a, const Extent& b) { return a.ptr == b.ptr; }), all.end());
  return all;
}

// every device pointer of a version lies in one of its own extents, and every extent in a slab of the store
int check_version(StoredBatch& b, const std::vector<Arena::Slab>& slabs) {
  std::vector<Extent> own = b.extents;
  std::sort(own.begin(), own.end(), by_ptr);
  for (const Extent& e : own)
    if (slab_of(slabs, e.ptr) < 0 || slab_of(slabs, e.ptr + e.bytes - 1) != slab_of(slabs, e.ptr))
      return set_error(SD_ERR_STATE, "sd_store_reclaim: batch %lld: an extent of %zu bytes lies outside the store's slabs", (long long)b.batch_id, e.bytes);
  int bad_col = 0;
  const char* bad = nullptr;
  uintptr_t bad_addr = 0;
  visit_device_pointers(b, [&](uintptr_t a, int col, const char* what) {
    if (!bad && !containing(own, a)) { bad = what; bad_col = col; bad_addr = a; }
    return a;
  });
  if (bad)
    return set_error(SD_ERR_STATE, "sd_store_reclaim: batch %lld column %d: %s (0x%llx) lies in no extent of its version; nothing was moved",
                     (long long)b.batch_id, bad_col, bad, (unsigned long long)bad_addr);
  return 0;
}

struct Move { uint8_t* src; size_t bytes; uint8_t* dst; };

struct StreamGuard {
  cudaStream_t st = nullptr;
  cudaEvent_t ev[3] = {};
  ~StreamGuard() {
    if (st) cudaStreamSynchronize(st);
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
    if (st) cudaStreamDestroy(st);
  }
};

// free the slabs of `pending` (base addresses) that hold no extent of a current version or of a retired version an open
// scan may read; the others stay pending
int free_unreadable(sd_store* s, std::vector<uint8_t*>& pending, int64_t out[4]) {
  const auto t = std::chrono::steady_clock::now();
  std::vector<Arena::Slab> gone;
  {
    std::lock_guard<std::mutex> lock(s->mu);
    drop_unreadable_retired(s);
    const std::vector<Extent> live = live_extents(s, true);
    std::vector<uint8_t*> keep;
    for (uint8_t* base : pending) {
      size_t i = 0;
      while (i < s->arena.slabs.size() && s->arena.slabs[i].base != base) i++;
      if (i == s->arena.slabs.size()) continue;
      const Arena::Slab& sl = s->arena.slabs[i];
      auto it = std::lower_bound(live.begin(), live.end(), base, [](const Extent& e, const uint8_t* x) { return e.ptr < x; });
      if (it != live.end() && it->ptr < sl.base + sl.bytes) { keep.push_back(base); continue; }
      gone.push_back(s->arena.detach_slab(i));
    }
    pending.swap(keep);
  }
  for (const Arena::Slab& sl : gone) {   // (outside the lock: a cudaFree waits for the device)
    Arena::free_slab(s->device, sl);
    out[0]++;
    out[1] += (int64_t)sl.bytes;
  }
  SD_CUDA(cudaGetLastError());
  g_timing.free_ms += ms_since(t);
  return 0;
}

// one round: move the current versions' extents that lie in `sources` ([base, bytes) of slabs), install the new versions
// (the versions in `cur` are replaced only by this call: the store's mutate_mu is held)
int run_round(sd_store* s, cudaStream_t st, cudaEvent_t* ev, const std::vector<std::pair<uint8_t*, size_t>>& sources,
              std::vector<StoredBatch*>& cur, int64_t* moved) {
  // ---- what moves: per batch, its extents in the sources plus the extents of its DevDelta structs ----------------------
  std::map<size_t, std::vector<Move>> moves;   // by index in `cur`
  for (size_t bi = 0; bi < cur.size(); bi++)
    for (const Extent& e : cur[bi]->extents)
      for (const auto& src : sources)
        if (e.ptr >= src.first && e.ptr < src.first + src.second) { moves[bi].push_back(Move{e.ptr, e.bytes, nullptr}); break; }
  if (moves.empty()) return 0;
  for (auto& m : moves) {
    const StoredBatch& b = *cur[m.first];
    std::vector<Extent> own = b.extents;
    std::sort(own.begin(), own.end(), by_ptr);
    for (const StoredCol& c : b.cols)
      for (int d = 0; d < 2; d++) {
        if (!c.present || !c.delta[d].present || !c.dev_delta[d]) continue;
        const Extent* e = containing(own, (uintptr_t)c.dev_delta[d]);
        if (!e) return set_error(SD_ERR_STATE, "sd_store_reclaim: batch %lld: a DevDelta struct lies in no extent of its version", (long long)b.batch_id);
        bool have = false;
        for (const Move& mv : m.second) have = have || mv.src == e->ptr;
        if (!have) m.second.push_back(Move{e->ptr, e->bytes, nullptr});
      }
  }
  // ---- destinations: same address modulo 256 ---------------------------------------------------------------------------
  std::vector<CopyJob> jobs;
  std::vector<int64_t> first_chunk;
  int64_t nchunks = 0, bytes = 0;
  {
    std::lock_guard<std::mutex> lock(s->mu);
    for (auto& m : moves)
      for (Move& mv : m.second) {
        const size_t phase = (uintptr_t)mv.src & 255;
        mv.dst = s->arena.alloc(mv.bytes, 256, (256 - phase) & 255);
        if (!mv.dst) return SD_ERR_CUDA;
        jobs.push_back(CopyJob{mv.src, mv.dst, (int64_t)mv.bytes});
        first_chunk.push_back(nchunks);
        nchunks += ((int64_t)mv.bytes + CP_CHUNK - 1) / CP_CHUNK;
        bytes += (int64_t)mv.bytes;
      }
  }
  // ---- copy ---------------------------------------------------------------------------------------------------------------
  DevScratch ds;
  ds.st = st;
  CopyJob* d_jobs;
  int64_t* d_first;
  int rc;
  if ((rc = ds.get(&d_jobs, sizeof(CopyJob) * jobs.size())) || (rc = ds.get(&d_first, 8 * first_chunk.size()))) return rc;
  // (pageable sources: staged before the calls return)
  SD_CUDA(cudaMemcpyAsync(d_jobs, jobs.data(), sizeof(CopyJob) * jobs.size(), cudaMemcpyHostToDevice, st));
  SD_CUDA(cudaMemcpyAsync(d_first, first_chunk.data(), 8 * first_chunk.size(), cudaMemcpyHostToDevice, st));
  static int ctas_per_sm = -1, num_sms = 0;
  if (ctas_per_sm < 0) {
    SD_CUDA(cudaFuncSetAttribute(reclaim_copy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CP_SMEM));
    SD_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas_per_sm, reclaim_copy_kernel, CP_THREADS, CP_SMEM));
    SD_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, s->device));
  }
  const int64_t grid = std::min<int64_t>(nchunks, (int64_t)std::max(1, ctas_per_sm) * std::max(1, num_sms));
  SD_CUDA(cudaEventRecord(ev[0], st));
  reclaim_copy_kernel<<<(unsigned)grid, CP_THREADS, CP_SMEM, st>>>(d_jobs, d_first, (int)jobs.size(), nchunks);
  SD_CUDA(cudaGetLastError());
  SD_CUDA(cudaEventRecord(ev[1], st));
  // ---- new versions: rebased pointers, rebased DevDelta structs written over their copies -------------------------------
  const auto t_inst = std::chrono::steady_clock::now();
  FreshBatches fresh;
  std::vector<std::pair<size_t, StoredBatch*>> installed;
  for (auto& m : moves) {
    std::vector<Move>& mv = m.second;
    std::sort(mv.begin(), mv.end(), [](const Move& a, const Move& b) { return a.src < b.src; });
    const StoredBatch& old = *cur[m.first];
    std::unique_ptr<StoredBatch> nb(new StoredBatch(old));
    nb->uid = next_batch_uid();
    auto rebase = [&](uintptr_t a) -> uintptr_t {
      auto it = std::upper_bound(mv.begin(), mv.end(), a, [](uintptr_t x, const Move& y) { return x < (uintptr_t)y.src; });
      if (it == mv.begin()) return a;
      --it;
      return a < (uintptr_t)it->src + it->bytes ? (uintptr_t)it->dst + (a - (uintptr_t)it->src) : a;
    };
    visit_device_pointers(*nb, [&](uintptr_t a, int, const char*) { return rebase(a); });
    for (Extent& e : nb->extents) e.ptr = reinterpret_cast<uint8_t*>(rebase((uintptr_t)e.ptr));
    for (StoredCol& c : nb->cols)
      for (int d = 0; d < 2; d++)
        if (c.present && c.delta[d].present && c.dev_delta[d])
          SD_CUDA(cudaMemcpyAsync(c.dev_delta[d], &c.delta[d].dev, sizeof(DevDelta), cudaMemcpyHostToDevice, st));
    installed.emplace_back(m.first, nb.get());
    fresh.emplace_back(&old, std::move(nb));
  }
  SD_CUDA(cudaStreamSynchronize(st));   // the new bytes are in place before any scan can see them
  float ms = 0;
  cudaEventElapsedTime(&ms, ev[0], ev[1]);
  g_timing.copy_ms += ms;
  if ((rc = store_install(s, fresh, {}, "sd_store_reclaim"))) return rc;
  for (auto& i : installed) cur[i.first] = i.second;
  *moved += bytes;
  g_timing.install_ms += ms_since(t_inst);
  return 0;
}

int reclaim(sd_store* s, double max_live_fraction, int64_t out[4]) {
  const auto t0 = std::chrono::steady_clock::now();
  if (!s || !out) return set_error(SD_ERR_INVALID, "sd_store_reclaim: null argument");
  if (!(max_live_fraction >= 0.0 && max_live_fraction <= 1.0))
    return set_error(SD_ERR_INVALID, "sd_store_reclaim: max_live_fraction must lie in [0, 1] (got %g)", max_live_fraction);
  std::lock_guard<std::mutex> serial(s->mutate_mu);   // no UPDATE / DELETE / compaction meanwhile
  std::lock_guard<std::mutex> encoder(s->enc_mu);     // nor a device encode writing bytes of a batch not yet published
  g_timing = Timing();
  for (int q = 0; q < 4; q++) out[q] = 0;
  SD_CUDA(cudaSetDevice(s->device));
  StreamGuard sg;
  SD_CUDA(cudaStreamCreateWithFlags(&sg.st, cudaStreamNonBlocking));
  for (cudaEvent_t& e : sg.ev) SD_CUDA(cudaEventCreate(&e));
  // ---- inventory + selection under the store's lock ------------------------------------------------------------------------
  std::vector<StoredBatch*> cur;
  std::vector<uint8_t*> pending;                    // slabs to free once no open scan can read them
  struct Evac { double fraction; uint8_t* base; size_t bytes; };
  std::vector<Evac> evac;                           // the slabs to empty
  {
    std::lock_guard<std::mutex> lock(s->mu);
    int rc = store_flush_lz4(s);   // pending expansions write into the slabs: finish them first
    if (rc) return rc;
    if ((rc = store_lz4_check(s))) return rc;
    SD_CUDA(cudaEventRecord(sg.ev[2], s->copy_stream));   // ... and the uploads still in flight
    SD_CUDA(cudaStreamWaitEvent(sg.st, sg.ev[2], 0));
    for (int q = 0; q + 1 < s->num_copy_streams; q++) {
      SD_CUDA(cudaEventRecord(s->extra_done[q], s->extra_streams[q]));
      SD_CUDA(cudaStreamWaitEvent(sg.st, s->extra_done[q], 0));
    }
    std::vector<Arena::Slab> slabs = s->arena.slabs;
    std::sort(slabs.begin(), slabs.end(), [](const Arena::Slab& a, const Arena::Slab& b) { return a.base < b.base; });
    for (auto& b : s->batches)
      if ((rc = check_version(*b, slabs))) return rc;
    s->arena.close_slab();   // new allocations (this call's destinations, concurrent puts) go to fresh slabs
    drop_unreadable_retired(s);
    for (auto& b : s->batches) cur.push_back(b.get());
    std::vector<size_t> live(slabs.size(), 0);
    for (const Extent& e : live_extents(s, true)) {
      const int k = slab_of(slabs, e.ptr);
      if (k >= 0) live[(size_t)k] += e.bytes;
    }
    for (size_t k = 0; k < slabs.size(); k++) {
      if (live[k] == 0) pending.push_back(slabs[k].base);
      else if ((double)live[k] <= max_live_fraction * (double)slabs[k].bytes)
        evac.push_back(Evac{(double)live[k] / (double)slabs[k].bytes, slabs[k].base, slabs[k].bytes});
    }
  }
  std::stable_sort(evac.begin(), evac.end(), [](const Evac& a, const Evac& b) { return a.fraction < b.fraction; });
  g_timing.plan_ms = ms_since(t0);
  int rc = free_unreadable(s, pending, out);   // slabs nothing lives in: no copy
  if (rc) return rc;
  // ---- rounds: sources in ascending live fraction while their current extents fit one destination slab -----------------
  size_t next = 0;
  int round = 0;
  while (next < evac.size()) {
    std::vector<std::pair<uint8_t*, size_t>> sources;
    size_t fill = 0;
    for (; next < evac.size(); next++) {
      const std::pair<uint8_t*, size_t> src(evac[next].base, evac[next].bytes);
      size_t need = 0;
      for (StoredBatch* b : cur)
        for (const Extent& e : b->extents)
          if (e.ptr >= src.first && e.ptr < src.first + src.second) need += e.bytes + 256;
      if (!sources.empty() && fill + need > s->arena.slab_bytes) break;
      sources.push_back(src);
      fill += need;
    }
    rc = run_round(s, sg.st, sg.ev, sources, cur, &out[2]);
    if (rc) {
      const std::string why = last_error_cstr();
      return set_error(rc, "sd_store_reclaim: round %d failed and installed nothing (%d earlier rounds stay installed; their bytes are identical): %s",
                       round + 1, round, why.c_str());
    }
    round++;
    g_timing.rounds = round;
    for (const auto& src : sources) pending.push_back(src.first);
    if ((rc = free_unreadable(s, pending, out))) return rc;
  }
  out[3] = (int64_t)pending.size();
  g_timing.total_ms = ms_since(t0);
  return 0;
}

}  // namespace
}  // namespace sd

extern "C" {

int sd_store_reclaim(sd_store* s, double max_live_fraction, int64_t out[4]) { return sd::reclaim(s, max_live_fraction, out); }

// the calling thread's last sd_store_reclaim: [0] inventory + planning ms (host) [1] copy ms (device events) [2] install ms
// [3] free ms [4] whole call ms (host clock) [5] rounds
int sdx_last_reclaim_timing(double out[6]) {
  const sd::Timing& t = sd::g_timing;
  out[0] = t.plan_ms; out[1] = t.copy_ms; out[2] = t.install_ms; out[3] = t.free_ms; out[4] = t.total_ms; out[5] = t.rounds;
  return 0;
}

// bytes of the extents of the current batch versions ([0]) and of the retired versions still kept for open scans that the
// current ones do not share ([1])
int sdx_store_extent_bytes(sd_store* s, int64_t out[2]) {
  if (!s || !out) return sd::set_error(SD_ERR_INVALID, "sdx_store_extent_bytes: null argument");
  std::lock_guard<std::mutex> lock(s->mu);
  int64_t cur = 0, all = 0;
  for (const sd::Extent& e : sd::live_extents(s, false)) cur += (int64_t)e.bytes;
  for (const sd::Extent& e : sd::live_extents(s, true)) all += (int64_t)e.bytes;
  out[0] = cur;
  out[1] = all - cur;
  return 0;
}

}  // extern "C"
