// sd_compact.cu -- compaction of resident batches on the device: the update deltas and delete masks that UPDATE / DELETE leave
// behind (sd_mutate.cu) are folded back into the base columns, so later scans take the staged fast path again instead of the
// overlay path.  The result of a rewritten column is, byte for byte, what ingest (sd_store_encode_batch) writes for the
// batch's live rows with their current values -- the reference's ColumnDeltaEncoder.merge into a full column
// (enc/ColumnDeltaEncoder.scala:348-556; sd_delta_merge with existing_is_delta = 0 is its host restatement) with the deleted
// rows dropped.
//
// One pass over the selected batches, batched across all of them, in rounds whose scratch stays under ROUND_SCRATCH:
//   1. materialise  one CTA per (batch, rewritten column), tiles of 1024 rows: every live row's current value (base decoded
//                   with the scan's own helpers, then depth 1, then depth 0 -- depth 0 wins) and null flag, written at the
//                   row's live rank.  STRING columns travel as codes of the batch's unified code space, mapped on the host
//                   to one canonical code per distinct string; an atomicMin of the live rank per code finds the first-seen
//                   order of the dictionary without moving string bytes;
//   2. encode       the encoder of sd_encode.cu (null words, one feedback read-back, layout in the store's arena through
//                   store_register_encoded, one write launch for every column of the round);
//   3. install      every new batch version and the removal of fully deleted batches in one hold of the store's lock.
#include <algorithm>
#include <chrono>
#include <climits>
#include <cstdlib>
#include <cstring>
#include <unordered_map>

#include "sd_host.h"
#include "sd_kernels.cuh"

namespace sd {
namespace {

constexpr int CT = 1024;                              // threads of the materialise kernel = rows per tile
constexpr size_t ROUND_SCRATCH = size_t(2) << 30;     // device scratch of one round (materialised values + encoder state);
                                                      // SD_TUNE_COMPACT_ROUND_BYTES overrides it (tests: many rounds)
constexpr int32_t NOT_SEEN = 0x7f7f7f7f;              // first_seen of a code no live row holds (memset byte 0x7f)

struct MatJob {
  DevCol col;                 // the base column with its delta pointers
  const int32_t* deletes;     // ascending deleted ordinals of the batch, or nullptr
  const int32_t* canon;       // STRING: unified code -> canonical code
  int32_t* first_seen;        // STRING: canonical code -> smallest live rank that holds it
  uint8_t* out_vals;          // the live rows' values at their rank (the type's width; STRING: int32 canonical code)
  uint8_t* out_nulls;         // the live rows' null flags
  int32_t num_rows;
  int32_t num_deletes;
  int32_t kind;
  int32_t pad_;
};

template <int K>
__device__ void materialise(const MatJob& j) {
  typedef typename KindT<K>::T T;
  const DevCol& c = j.col;
  for (int i = threadIdx.x; i < j.num_rows; i += CT) {
    int rank = i;
    if (j.num_deletes) {   // live rank = ordinal - deleted rows before it
      const int q = lower_bound_i32(j.deletes, 0, j.num_deletes, i);
      if (q < j.num_deletes && j.deletes[q] == i) continue;
      rank = i - q;
    }
    bool isnull = false, found = false;
    T v = (T)0;
    // the depth-0 delta wins on an equal position, then depth 1 (enc/UpdatedColumnDecoder.scala:95-104)
    for (int depth = 0; depth < 2 && !found; depth++) {
      const DevDelta* d = depth ? c.delta1 : c.delta0;
      if (!d || d->n == 0) continue;
      const int q = lower_bound_i32(d->positions, 0, d->n, i);
      if (q < d->n && d->positions[q] == i) { v = delta_value_at<K>(d, q, c.dict_n, &isnull); found = true; }
    }
    if (!found) {   // base value #(ordinal - nulls before it), the nulls counted from the host prefix per 512 rows
      int64_t k = i;
      if (c.nulls) {
        const int w = i >> 6;
        const uint64_t word = w < c.nwords ? c.nulls[w] : 0ull;
        isnull = (word >> (i & 63)) & 1ull;
        int before = c.tile_nulls ? c.tile_nulls[i / NULL_PREFIX_ROWS] : 0;
        for (int x = (i / NULL_PREFIX_ROWS) * NULL_PREFIX_WORDS; x < w && x < c.nwords; x++) before += __popcll(c.nulls[x]);
        k = i - (before + __popcll(word & ((1ull << (i & 63)) - 1ull)));
      }
      if (!isnull) v = decode_value_any<K>(c.data, c.dict, c.run_ends, c.enc, c.nruns, k);
    }
    j.out_nulls[rank] = isnull ? 1 : 0;
    if (K == K_CODE) {
      const int32_t code = isnull ? 0 : j.canon[(int)v];
      reinterpret_cast<int32_t*>(j.out_vals)[rank] = code;
      // one atomic per code and thread while it can still lower the minimum: the columns of a batch hold few distinct
      // strings, and an atomic per row onto the same few addresses serialises the whole CTA
      if (!isnull && rank < *reinterpret_cast<volatile int32_t*>(j.first_seen + code)) atomicMin(j.first_seen + code, rank);
    } else {
      reinterpret_cast<T*>(j.out_vals)[rank] = isnull ? (T)0 : v;
    }
  }
}

__global__ void __launch_bounds__(CT) materialise_kernel(const MatJob* jobs) {
  const MatJob& j = jobs[blockIdx.x];
  switch (j.kind) {
    case K_I8: materialise<K_I8>(j); break;
    case K_I16: materialise<K_I16>(j); break;
    case K_I32: materialise<K_I32>(j); break;
    case K_I64: materialise<K_I64>(j); break;
    case K_F32: materialise<K_F32>(j); break;
    case K_F64: materialise<K_F64>(j); break;
    case K_BOOL: materialise<K_BOOL>(j); break;
    default: materialise<K_CODE>(j); break;
  }
}

int value_width(int t) {   // bytes of one materialised value
  switch (t) {
    case SD_BOOLEAN: case SD_BYTE: return 1;
    case SD_SHORT: return 2;
    case SD_INT: case SD_DATE: case SD_FLOAT: case SD_STRING: return 4;
    default: return 8;
  }
}

// one rewritten column of a selected batch
struct ColWork {
  int table_col = 0;
  std::vector<int32_t> canon;          // STRING: unified code -> canonical code
  std::vector<std::string> canon_str;  // STRING: canonical code -> its string
  size_t off_vals = 0, off_nulls = 0, off_words = 0, off_codes = 0, off_slot = 0, off_pairs = 0;
  EncJob job;
};
struct BatchWork {
  const StoredBatch* b = nullptr;
  int n_live = 0;
  std::vector<ColWork> cols;
  size_t scratch = 0;
};

inline size_t up256(size_t x) { return (x + 255) & ~size_t(255); }

size_t plan_scratch(BatchWork& bw) {
  size_t total = 0;
  for (ColWork& cw : bw.cols) {
    const size_t n = (size_t)bw.n_live;
    total += up256(n * value_width(cw.job.type) + 64) + up256(n + 64) + up256((n + 63) / 64 * 8 + 64) + 128;
    total += up256(cw.canon.size() * 4 + 64) * 3 + up256(cw.canon.size() * 8 + 64);
  }
  return total;
}

struct Timing { double mat_ms = 0, enc_ms = 0, host_ms = 0, total_ms = 0, rows = 0, bytes = 0; };
thread_local Timing g_timing;

uint8_t* scratch_alloc(void* ctx, size_t bytes) {
  uint8_t* p = nullptr;
  return reinterpret_cast<DevScratch*>(ctx)->get(&p, bytes) ? nullptr : p;
}

struct StreamGuard {
  cudaStream_t st = nullptr;
  cudaEvent_t ev[6] = {};
  ~StreamGuard() {
    if (st) cudaStreamSynchronize(st);
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
    if (st) cudaStreamDestroy(st);
  }
};

// one round: materialise + encode the columns of `round`, new batch versions into `fresh`
int compact_round(sd_store* s, cudaStream_t st, cudaEvent_t* ev, std::vector<BatchWork*>& round, FreshBatches& fresh, int64_t* written) {
  std::vector<ColWork*> cws;
  for (BatchWork* bw : round) for (ColWork& cw : bw->cols) cws.push_back(&cw);
  const size_t nj = cws.size();
  // ---- scratch: one allocation per kind of buffer, carved per column ---------------------------------------------------
  size_t vals = 0, nulls = 0, words = 0, codes = 0, slot = 0, pairs = 0;
  for (BatchWork* bw : round) {
    const size_t n = (size_t)bw->n_live;
    for (ColWork& cw : bw->cols) {
      cw.off_vals = vals; vals += up256(n * value_width(cw.job.type) + 64);
      cw.off_nulls = nulls; nulls += up256(n + 64);
      cw.off_words = words; words += up256((n + 63) / 64 * 8 + 64);
      cw.off_codes = codes; codes += cw.canon.size();
      cw.off_slot = slot; slot += cw.canon.size();
      cw.off_pairs = pairs; pairs += cw.canon.size();
    }
  }
  DevScratch ds;
  ds.st = st;
  PinnedArena pin;
  uint8_t *d_vals, *d_nulls, *d_words, *d_fbst;
  int32_t *d_canon, *d_first, *d_slot;
  int2* d_pairs;
  MatJob* d_jobs;
  int rc;
  if ((rc = ds.get(&d_vals, vals)) || (rc = ds.get(&d_nulls, nulls)) || (rc = ds.get(&d_words, words)) || (rc = ds.get(&d_fbst, 128 * nj)) ||
      (rc = ds.get(&d_canon, 4 * codes + 16)) || (rc = ds.get(&d_first, 4 * codes + 16)) || (rc = ds.get(&d_slot, 4 * slot + 16)) ||
      (rc = ds.get(&d_pairs, 8 * pairs + 16)) || (rc = ds.get(&d_jobs, sizeof(MatJob) * nj)))
    return rc;
  SD_CUDA(cudaMemsetAsync(d_fbst, 0, 128 * nj, st));
  if (codes) SD_CUDA(cudaMemsetAsync(d_first, 0x7f, 4 * codes, st));
  // ---- materialise ---------------------------------------------------------------------------------------------------------
  std::vector<MatJob> mj(nj);
  std::vector<int32_t> h_canon;
  h_canon.reserve(codes);
  size_t k = 0;
  for (BatchWork* bw : round) {
    for (ColWork& cw : bw->cols) {
      const StoredCol& col = bw->b->cols[cw.table_col];
      MatJob& m = mj[k++];
      memset(&m, 0, sizeof(m));
      m.col = col.dev;
      m.col.delta0 = col.delta[0].present ? col.dev_delta[0] : nullptr;
      m.col.delta1 = col.delta[1].present ? col.dev_delta[1] : nullptr;
      m.deletes = bw->b->num_deletes ? bw->b->dev_deletes : nullptr;
      m.num_deletes = bw->b->num_deletes;
      m.num_rows = bw->b->num_rows;
      m.kind = kind_of_type(cw.job.type);
      m.out_vals = d_vals + cw.off_vals;
      m.out_nulls = d_nulls + cw.off_nulls;
      if (!cw.canon.empty()) {
        m.canon = d_canon + cw.off_codes;
        m.first_seen = d_first + cw.off_codes;
        h_canon.insert(h_canon.end(), cw.canon.begin(), cw.canon.end());
      }
      EncJob& j = cw.job;
      j.n = bw->n_live;
      j.d_values = m.out_vals;
      j.d_nulls = j.nullable ? m.out_nulls : nullptr;
      j.d_words = reinterpret_cast<uint64_t*>(d_words + cw.off_words);
      j.d_fb = reinterpret_cast<int*>(d_fbst + 128 * (k - 1));
      j.d_stat = reinterpret_cast<uint64_t*>(d_fbst + 128 * (k - 1) + 64);
      if (j.type == SD_STRING) { j.d_slot_code = d_slot + cw.off_slot; j.d_slot_pairs = d_pairs + cw.off_pairs; }
    }
  }
  uint8_t* h_jobs = pin.alloc(sizeof(MatJob) * nj + h_canon.size() * 4);
  if (!h_jobs) return SD_ERR_CUDA;
  memcpy(h_jobs, mj.data(), sizeof(MatJob) * nj);
  SD_CUDA(cudaMemcpyAsync(d_jobs, h_jobs, sizeof(MatJob) * nj, cudaMemcpyHostToDevice, st));
  if (!h_canon.empty()) {
    memcpy(h_jobs + sizeof(MatJob) * nj, h_canon.data(), h_canon.size() * 4);
    SD_CUDA(cudaMemcpyAsync(d_canon, h_jobs + sizeof(MatJob) * nj, h_canon.size() * 4, cudaMemcpyHostToDevice, st));
  }
  SD_CUDA(cudaEventRecord(ev[0], st));
  if (nj) {
    materialise_kernel<<<(unsigned)nj, CT, 0, st>>>(d_jobs);
    SD_CUDA(cudaGetLastError());
  }
  SD_CUDA(cudaEventRecord(ev[1], st));
  std::vector<EncJob*> jobs;
  for (ColWork* cw : cws) jobs.push_back(&cw->job);
  if ((rc = enc_null_words_many(st, jobs, scratch_alloc, &ds, pin))) return rc;
  SD_CUDA(cudaEventRecord(ev[2], st));
  // ---- one feedback read-back: null counts / trimmed word counts, first-seen ranks of the codes ---------------------------
  std::vector<int32_t> fbst(32 * nj), first(codes);
  SD_CUDA(cudaMemcpyAsync(fbst.data(), d_fbst, 128 * nj, cudaMemcpyDeviceToHost, st));
  if (codes) SD_CUDA(cudaMemcpyAsync(first.data(), d_first, 4 * codes, cudaMemcpyDeviceToHost, st));
  SD_CUDA(cudaStreamSynchronize(st));
  for (size_t q = 0; q < nj; q++) {
    EncJob& j = cws[q]->job;
    j.fb[0] = fbst[32 * q]; j.fb[1] = fbst[32 * q + 1];
    if (j.type == SD_STRING) {   // dictionary in first-seen order: the codes some live row holds, by their first rank
      std::vector<int2> seen;
      for (size_t c = 0; c < cws[q]->canon.size(); c++) {
        const int32_t r = first[cws[q]->off_codes + c];
        if (r != NOT_SEEN) seen.push_back(make_int2((int)c, r));
      }
      const std::vector<std::string>& strs = cws[q]->canon_str;
      enc_first_seen_dict(j, seen, [&](int code, int) { return strs[(size_t)code]; });
    }
  }
  const bool any_words = enc_queue_words(st, jobs, &rc);   // the trimmed null words (only columns that hold NULLs)
  if (rc) return rc;
  if (any_words) SD_CUDA(cudaStreamSynchronize(st));
  // ---- layout of every column of the round in the store's arena; new batch versions --------------------------------------
  const auto t_host = std::chrono::steady_clock::now();
  std::vector<std::unique_ptr<StoredBatch>> nbs;
  std::vector<std::vector<ColStat>> stats(round.size());   // per batch: the entries of its rewritten columns
  std::vector<ColStat*> job_stats;
  {
    std::lock_guard<std::mutex> lock(s->mu);
    const size_t used0 = s->arena.used;
    for (size_t r = 0; r < round.size(); r++) {
      const StoredBatch& old = *round[r]->b;
      std::unique_ptr<StoredBatch> nb(new StoredBatch(old));
      nb->uid = next_batch_uid();
      nb->num_rows = round[r]->n_live;
      nb->dev_deletes = nullptr; nb->num_deletes = 0; nb->has_deltas = false; nb->gone = false;
      stats[r].resize(round[r]->cols.size());
      ExtentRecorder rec(s->arena, &nb->extents);   // (the rewritten columns' old extents are pruned at install)
      for (size_t q = 0; q < round[r]->cols.size(); q++) {
        ColWork& cw = round[r]->cols[q];
        if ((rc = enc_layout(s, st, pin, cw.job, nb->cols[cw.table_col], stats[r][q]))) return rc;
        job_stats.push_back(&stats[r][q]);
      }
      nbs.push_back(std::move(nb));
    }
    *written += (int64_t)(s->arena.used - used0);
    // the side uploads of the layout (null words, "nulls before" prefixes) went over the store's copy stream
    SD_CUDA(cudaEventRecord(ev[5], s->copy_stream));
    SD_CUDA(cudaStreamWaitEvent(st, ev[5], 0));
  }
  g_timing.host_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_host).count();
  if ((rc = enc_write(st, scratch_alloc, &ds, pin, jobs, job_stats, ev[3], ev[4]))) return rc;
  SD_CUDA(cudaStreamSynchronize(st));
  float a = 0, b = 0, c = 0;
  cudaEventElapsedTime(&a, ev[0], ev[1]);
  cudaEventElapsedTime(&b, ev[1], ev[2]);
  cudaEventElapsedTime(&c, ev[3], ev[4]);
  g_timing.mat_ms += a;
  g_timing.enc_ms += b + c;
  {   // scan images of the rewritten columns (the kept ones keep theirs)
    std::vector<StoredBatch*> fresh_nbs;
    for (auto& nb : nbs) fresh_nbs.push_back(nb.get());
    if ((rc = build_images(s, st, fresh_nbs, false))) return rc;
  }
  for (size_t r = 0; r < round.size(); r++) {   // the rewritten columns' entries replace theirs; every other entry is kept as it is
    std::vector<std::pair<int, const ColStat*>> repl;
    for (size_t q = 0; q < round[r]->cols.size(); q++) repl.emplace_back(round[r]->cols[q].table_col, &stats[r][q]);
    if (nbs[r]->stats.empty()) {   // the batch had no stats row: one with the rewritten columns' entries
      std::vector<ColStat> all(s->schema.size());
      for (auto& e : repl) all[(size_t)e.first] = *e.second;
      nbs[r]->stats = stats_row_bytes(round[r]->n_live, all);
      nbs[r]->stats_ncols = (int32_t)s->schema.size();
    } else {
      stats_row_replace(nbs[r]->stats, nbs[r]->stats_ncols, round[r]->n_live, repl);
    }
    fresh.emplace_back(round[r]->b, std::move(nbs[r]));
  }
  return 0;
}

int compact(sd_store* s, const int32_t* bucket_ids, int32_t nbuckets, double min_dirty_fraction, int64_t out[4]) {
  const auto t0 = std::chrono::steady_clock::now();
  if (!s || !out) return set_error(SD_ERR_INVALID, "sd_store_compact: null argument");
  if (!(min_dirty_fraction >= 0)) return set_error(SD_ERR_INVALID, "sd_store_compact: min_dirty_fraction must be >= 0 (got %g)", min_dirty_fraction);
  if (nbuckets < 0 || (nbuckets > 0 && !bucket_ids)) return set_error(SD_ERR_INVALID, "sd_store_compact: bad bucket list");
  std::lock_guard<std::mutex> serial(s->mutate_mu);   // serialised with UPDATE / DELETE on this store
  g_timing = Timing();
  for (int q = 0; q < 4; q++) out[q] = 0;
  SD_CUDA(cudaSetDevice(s->device));
  StreamGuard sg;
  SD_CUDA(cudaStreamCreateWithFlags(&sg.st, cudaStreamNonBlocking));
  for (cudaEvent_t& e : sg.ev) SD_CUDA(cudaEventCreate(&e));
  cudaStream_t st = sg.st;
  // ---- the batches present now; their bytes (uploads, LZ4 expansions) complete before the compaction reads them ----------
  std::vector<const StoredBatch*> snap;
  {
    std::lock_guard<std::mutex> lock(s->mu);
    int rc = store_flush_lz4(s);   // expand what is pending and refuse a corrupt payload, as a scan does
    if (rc) return rc;
    if ((rc = store_lz4_check(s))) return rc;
    SD_CUDA(cudaEventRecord(sg.ev[5], s->copy_stream));
    SD_CUDA(cudaStreamWaitEvent(st, sg.ev[5], 0));
    for (int q = 0; q + 1 < s->num_copy_streams; q++) {
      SD_CUDA(cudaEventRecord(s->extra_done[q], s->extra_streams[q]));
      SD_CUDA(cudaStreamWaitEvent(st, s->extra_done[q], 0));
    }
    for (auto& b : s->batches) {
      bool in = nbuckets == 0;
      for (int q = 0; q < nbuckets && !in; q++) in = bucket_ids[q] == b->bucket_id;
      if (in) snap.push_back(b.get());
    }
  }
  // ---- selection -------------------------------------------------------------------------------------------------------
  std::vector<BatchWork> work;
  std::vector<const StoredBatch*> remove;
  for (const StoredBatch* b : snap) {
    const bool mask = b->dev_deletes != nullptr;
    int64_t dirty = mask ? b->num_deletes : 0;
    bool any_delta = false;
    for (const StoredCol& c : b->cols) {
      if (!c.present) continue;
      for (int d = 0; d < 2; d++) if (c.delta[d].present) { dirty += c.delta[d].dev.n; any_delta = true; }
    }
    if (!mask && !any_delta) continue;
    if ((double)dirty < min_dirty_fraction * (double)b->num_rows) continue;
    if (b->gone || (mask && b->num_deletes >= b->num_rows)) {   // every row deleted: the batch leaves the store
      remove.push_back(b);
      out[2] += b->num_deletes;
      continue;
    }
    BatchWork bw;
    bw.b = b;
    bw.n_live = b->num_rows - (mask ? b->num_deletes : 0);
    for (int t = 0; t < (int)b->cols.size(); t++) {
      const StoredCol& c = b->cols[t];
      if (!c.present || (!mask && !c.delta[0].present && !c.delta[1].present)) continue;
      const int type = s->schema[t].type;
      if (!c.unsupported.empty())
        return set_error(SD_ERR_UNSUPPORTED, "sd_store_compact: batch %lld column %d: %s", (long long)b->batch_id, t, c.unsupported.c_str());
      if (wide_decimal(type, s->schema[t].precision))
        return set_error(SD_ERR_UNSUPPORTED, "sd_store_compact: batch %lld column %d: a DECIMAL wider than 18 digits is not re-encoded on the device",
                         (long long)b->batch_id, t);
      if (c.raw_str)
        return set_error(SD_ERR_UNSUPPORTED, "sd_store_compact: batch %lld column %d: an Uncompressed STRING column is not re-encoded on the device",
                         (long long)b->batch_id, t);
      if (!value_width(type) || kind_of_type(type) < 0)
        return set_error(SD_ERR_UNSUPPORTED, "sd_store_compact: batch %lld column %d: type %d", (long long)b->batch_id, t, type);
      ColWork cw;
      cw.table_col = t;
      cw.job.table_col = t; cw.job.type = type; cw.job.nullable = s->schema[t].nullable != 0;
      if (type == SD_STRING) {   // unified codes -> one canonical code per distinct string
        const size_t u = std::max(c.dict_strings.size(), (size_t)c.dev.dict_n + 1);
        cw.canon.assign(u, 0);
        std::unordered_map<std::string, int32_t> first;
        for (size_t q = 0; q < c.dict_strings.size(); q++) {
          auto it = first.emplace(c.dict_strings[q], (int32_t)cw.canon_str.size());
          if (it.second) cw.canon_str.push_back(c.dict_strings[q]);
          cw.canon[q] = it.first->second;
        }
        if (cw.canon_str.empty()) cw.canon_str.push_back(std::string());
      }
      g_timing.bytes += (double)c.len;
      for (int d = 0; d < 2; d++) if (c.delta[d].present) g_timing.bytes += (double)c.delta[d].len;
      bw.cols.push_back(std::move(cw));
    }
    if (mask) g_timing.bytes += 4.0 * b->num_deletes;
    g_timing.rows += b->num_rows;
    out[2] += mask ? b->num_deletes : 0;
    bw.scratch = plan_scratch(bw);
    work.push_back(std::move(bw));
  }
  // ---- rounds under the scratch budget; everything is installed together at the end ---------------------------------------
  FreshBatches fresh;
  size_t budget = ROUND_SCRATCH;
  if (const char* e = getenv("SD_TUNE_COMPACT_ROUND_BYTES")) { const long long v = atoll(e); if (v > 0) budget = (size_t)v; }
  for (size_t i = 0; i < work.size();) {
    std::vector<BatchWork*> round;
    size_t bytes = 0;
    while (i < work.size() && (round.empty() || bytes + work[i].scratch <= budget)) { bytes += work[i].scratch; round.push_back(&work[i++]); }
    int rc = compact_round(s, st, sg.ev, round, fresh, &out[3]);
    if (rc) return rc;
  }
  const auto t_inst = std::chrono::steady_clock::now();
  if (!fresh.empty() || !remove.empty()) {
    int rc = store_install(s, fresh, remove, "sd_store_compact");
    if (rc) return rc;
  }
  g_timing.host_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_inst).count();
  out[0] = (int64_t)work.size();
  out[1] = (int64_t)remove.size();
  g_timing.total_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  return 0;
}

}  // namespace
}  // namespace sd

extern "C" {

int sd_store_compact(sd_store* s, const int32_t* bucket_ids, int32_t nbuckets, double min_dirty_fraction, int64_t out[4]) {
  return sd::compact(s, bucket_ids, nbuckets, min_dirty_fraction, out);
}

// host clock and device times of the calling thread's last sd_store_compact (tools/mutation_bench.py):
// [0] materialise ms [1] encode ms (device events) [2] host layout + install ms [3] whole call ms [4] rows read [5] bytes read
int sdx_last_compaction_timing(double out[6]) {
  const sd::Timing& t = sd::g_timing;
  out[0] = t.mat_ms; out[1] = t.enc_ms; out[2] = t.host_ms; out[3] = t.total_ms; out[4] = t.rows; out[5] = t.bytes;
  return 0;
}

}  // extern "C"
