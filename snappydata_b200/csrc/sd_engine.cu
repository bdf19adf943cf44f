// sd_engine.cu -- plan handles: stats-row batch skipping, per-batch descriptor/table preparation,
// kernel launch, partial-row emission (the buffers themselves: sd_aggregate.cpp).  Host-side counterpart of
//   ColumnTableScan.doProduce batch loop        core/execution/columnar/ColumnTableScan.scala:518-599
//   ColumnTableScan.generateStatPredicate       core/execution/columnar/ColumnTableScan.scala:820-963
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <mutex>

#include "sd_aggregate.h"
#include "sd_host.h"

using namespace sd;

namespace {

thread_local int t_device = 0;

// ---- stats-row batch skipping (ColumnTableScan.generateStatPredicate, :820-963) -------------------
struct Tri { bool isnull; bool v; };
Tri tri_and(Tri a, Tri b) { if ((!a.isnull && !a.v) || (!b.isnull && !b.v)) return {false, false}; if (a.isnull || b.isnull) return {true, false}; return {false, true}; }
Tri tri_or(Tri a, Tri b) { if ((!a.isnull && a.v) || (!b.isnull && b.v)) return {false, true}; if (a.isnull || b.isnull) return {true, false}; return {false, false}; }
Tri tri_cmp(const HVal& a, const HVal& b, int t, bool le) {
  if (a.isnull || b.isnull) return {true, false};
  const int c = cmp_hval(a, b, t);
  return {false, le ? c <= 0 : c < 0};
}
HVal lit_val(const sd_literal& l, int t, bool wide_slot = false) {
  HVal v;
  v.isnull = l.is_null != 0;
  if (wide_slot) {   // a literal slot of a DECIMAL wider than 18 digits: its unscaled value as bytes
    if (!l.s || l.slen < 1 || l.slen > 16) v.isnull = true;   // (sd_plan_set_literals refuses such a value)
    else if (!v.isnull) v.w = dec_from_bytes(reinterpret_cast<const uint8_t*>(l.s), (size_t)l.slen);
    return v;
  }
  v.i = l.i;
  v.w = l.i;   // DECIMAL (precision <= 18): cmp_hval compares .w
  v.d = t == SD_FLOAT ? (double)(float)l.d : l.d;
  if (l.s && l.slen > 0) v.s.assign(l.s, (size_t)l.slen);
  return v;
}

struct StatEval {
  const PlanSpec& p;
  const std::vector<sd_literal>& lits;
  const uint8_t* stats; int64_t slen; int nfields; int num_rows;
  int node_col(int a, int b) const { return p.exprs[a].op == SD_OP_COL ? a : b; }
  static bool wide_ft(int ft) { return ft_base(ft) == SD_DECIMAL && ft_precision(ft) > 18; }
  bool stat(int ord, int which, int type, HVal* out) const {   // which: 0 lower, 1 upper, 2 nullCount
    const int idx = 1 + 3 * ord + which;
    return idx < nfields && unsafe_field(stats, slen, nfields, idx, which == 2 ? (int)SD_INT : type, out);
  }
  // true when a stats filter is defined for `node` (buildFilter.isDefinedAt)
  bool eval(int node, Tri* out) const {
    const sd_expr& e = p.exprs[node];
    Tri l, r;
    switch (e.op) {
      case SD_OP_AND: {
        const bool dl = eval(e.a, &l), dr = eval(e.b, &r);
        if (!dl && !dr) return false;
        *out = dl && dr ? tri_and(l, r) : (dl ? l : r);
        return true;
      }
      case SD_OP_OR: {
        const bool dl = eval(e.a, &l), dr = eval(e.b, &r);
        if (!(dl && dr)) return false;
        *out = tri_or(l, r);
        return true;
      }
      case SD_OP_EQ: case SD_OP_LT: case SD_OP_LE: case SD_OP_GT: case SD_OP_GE: {
        const sd_expr &ea = p.exprs[e.a], &eb = p.exprs[e.b];
        const bool cl = ea.op == SD_OP_COL && eb.op == SD_OP_LIT, cr = eb.op == SD_OP_COL && ea.op == SD_OP_LIT;
        if (!cl && !cr) return false;
        const sd_expr& ec = cl ? ea : eb;
        const sd_expr& el = cl ? eb : ea;
        const int t = ec.type, ord = p.cols[ec.a].table_ordinal;
        const int ft = field_type(t, t == SD_DECIMAL ? decimal_ps(p, node_col(e.a, e.b)) : 0);
        HVal lo, hi;
        if (!stat(ord, 0, wide_ft(ft) ? ft : t, &lo) || !stat(ord, 1, wide_ft(ft) ? ft : t, &hi)) return false;
        const HVal lit = lit_val(lits[el.a], wide_ft(ft) ? ft : t, p.lit_wide[(size_t)el.a] != 0);
        int op = e.op;
        if (cr) op = op == SD_OP_LT ? SD_OP_GT : op == SD_OP_LE ? SD_OP_GE : op == SD_OP_GT ? SD_OP_LT : op == SD_OP_GE ? SD_OP_LE : op;
        switch (op) {
          case SD_OP_EQ: *out = tri_and(tri_cmp(lo, lit, t, true), tri_cmp(lit, hi, t, true)); break;
          case SD_OP_LT: *out = tri_cmp(lo, lit, t, false); break;
          case SD_OP_LE: *out = tri_cmp(lo, lit, t, true); break;
          case SD_OP_GT: *out = tri_cmp(lit, hi, t, false); break;
          default: *out = tri_cmp(lit, hi, t, true); break;
        }
        return true;
      }
      case SD_OP_IN: {
        const sd_expr& ea = p.exprs[e.a];
        if (ea.op != SD_OP_COL || e.c > 200 || e.c < 1) return false;
        const int ord = p.cols[ea.a].table_ordinal;
        const int t = node_is_wide(p, e.a) ? field_type(SD_DECIMAL, decimal_ps(p, e.a)) : ea.type;
        HVal lo, hi, mn, mx;
        if (!stat(ord, 0, t, &lo) || !stat(ord, 1, t, &hi)) return false;
        bool have = false;
        for (int k = 0; k < e.c; k++) {   // Greatest / Least skip nulls
          if (lits[e.b + k].is_null) continue;
          const HVal v = lit_val(lits[e.b + k], t, p.lit_wide[(size_t)(e.b + k)] != 0);
          if (!have) { mn = mx = v; have = true; }
          else { if (cmp_hval(v, mn, t) < 0) mn = v; if (cmp_hval(v, mx, t) > 0) mx = v; }
        }
        if (!have) mn.isnull = mx.isnull = true;
        *out = tri_and(tri_cmp(lo, mx, t, true), tri_cmp(mn, hi, t, true));
        return true;
      }
      case SD_OP_STARTSWITH: {   // StartsWithForStats (ColumnTableScan.scala:1028-1088); never NULL
        const sd_expr &ea = p.exprs[e.a], &eb = p.exprs[e.b];
        if (ea.op != SD_OP_COL || eb.op != SD_OP_LIT) return false;
        const int ord = p.cols[ea.a].table_ordinal;
        HVal lo, hi;
        if (!stat(ord, 0, SD_STRING, &lo) || !stat(ord, 1, SD_STRING, &hi)) return false;
        const sd_literal& L = lits[eb.a];
        Tri r0 = {false, true};
        if (!L.is_null) {
          std::string pat(L.s ? L.s : "", (size_t)std::max(0, L.slen)), up = pat;
          int last = (int)up.size() - 1;
          while (last >= 0 && (uint8_t)up[last] == 0xff) last--;
          if (last < 0 || lo.isnull) {
            if (!hi.isnull) r0.v = cmp_str(pat, hi.s) <= 0;
          } else {
            up[last] = (char)((uint8_t)up[last] + 1);
            r0.v = (hi.isnull || cmp_str(pat, hi.s) <= 0) && cmp_str(lo.s, up) < 0;
          }
        }
        *out = r0;
        return true;
      }
      case SD_OP_ISNULL: case SD_OP_ISNOTNULL: {
        const sd_expr& ea = p.exprs[e.a];
        if (ea.op != SD_OP_COL) return false;
        HVal nc;
        if (!stat(p.cols[ea.a].table_ordinal, 2, SD_INT, &nc)) return false;
        *out = nc.isnull ? Tri{true, false} : Tri{false, e.op == SD_OP_ISNULL ? nc.i > 0 : num_rows > nc.i};
        return true;
      }
    }
    return false;
  }
};

}  // namespace

// batches of one launch per decode path: BATCH_ALL_FAST, BATCH_FAST_NULLS, BATCH_FAST_OVERLAY, general per-row decode
struct PathCounts {
  int32_t n[4] = {0, 0, 0, 0};
  // bytes of column values the launch reads: [0] every column verbatim, [1] scan images where the staged loads take them
  int64_t streamed[2] = {0, 0};
  // per scan column, the widest element any staged batch of the launch streams: [0] with verbatim values, [1] with scan
  // images where the batch has one; and the most img_tab words any batch's image of the column has
  uint8_t width[2][MAX_SCAN_COLS] = {};
  int32_t img_n[MAX_SCAN_COLS] = {};
};

// =====================================================================================================
struct sd_plan {
  int device = 0;
  PlanSpec spec;
  KernelEntry kernel;             // generic kernel of the plan
  KernelEntry kernel_reg;         // register-group-table variant (MODE_GROUPS, <= REG_GROUPS_MAX groups), lazily resolved
  int kernel_reg_state = 0;       // 0 unknown, 1 available, -1 unavailable
  // lazily resolved variants of the generic kernel, indexed by (NULL literal in this execution) | (scan has batches
  // that need the per-row decode / delta / delete paths) << 1; index 0 is `kernel` itself (staged paths only)
  KernelEntry variant[4];
  int variant_state[4] = {0, 0, 0, 0};
  bool force_hash = false;        // the dense group table was abandoned for the hash table during an execution
  const KernelEntry* active = nullptr;
  std::string kernel_name;
  int max_ctas_per_sm = 0;
  int chunk_rows = CHUNK_ROWS;
  size_t last_smem = (size_t)-1;
  const KernelEntry* last_kernel = nullptr;
  bool last_two_cta = false;      // last_kernel's two-CTA kernel was prepared
  int num_sms = 0;
  int smem_optin = 0;
  // literals
  std::vector<sd_literal> lits;
  std::vector<std::string> lit_strs;
  bool lits_set = false;
  // bytes of the STRING literals on the device (raw-string predicates compare against them); slot k: packed offset | length
  uint8_t* d_litpool = nullptr;
  size_t litpool_cap = 0;
  bool litpool_dirty = true;
  std::vector<int64_t> lit_packed;
  // streams / events
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  cudaEvent_t ev_start = nullptr, ev_stop = nullptr;
  // one event pair per launch of an execution: aggTime = the SUM of the launches' device times (host work between two
  // launches -- descriptor building, waiting for a store's lock -- is not kernel time)
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> ev_pairs;
  size_t ev_used = 0;
  // private store for sd_batch_submit / sd_rows_submit
  sd_store* priv = nullptr;
  // pending batches
  struct Pending { const StoredBatch* sb; };
  std::vector<Pending> pending;
  int64_t pending_bytes = 0;
  // device state
  Arena scratch;                 // descriptors, aux tables (reset per execution)
  // device state of one execution in ONE allocation so that it comes back in one copy:
  //   d_state = [8 x uint64 counters][result_cap x uint64 running result]
  uint64_t* d_state = nullptr;
  uint64_t* d_result = nullptr;  // = d_state + STATE_HDR
  uint64_t* h_pinned = nullptr;  // pinned host mirror of d_state: identities out, counters + result back
  size_t h_pinned_cap = 0;
  uint64_t* d_partials = nullptr;
  size_t partials_cap = 0;
  unsigned int* d_ticket = nullptr;
  unsigned long long* d_counters = nullptr;
  size_t result_cap = 0;         // entries
  int ngroups = 1;
  int32_t radix[MAX_KEYS] = {1, 1, 1, 1};
  bool result_init = false;
  // group key dictionaries (query-global ids per key column)
  std::vector<std::unordered_map<std::string, int>> key_ids;
  std::vector<std::vector<std::string>> key_vals;
  std::vector<int> key_null_id;
  // store-scan cache
  // A cached scan is a list of SEGMENTS, each a descriptor set over a run of the store's batches, launched one after the other
  // into the same result.  A store only ever appends batches (sd_store: never removed or moved), so when it has grown since
  // the last execution (ingest running beside the queries: BASELINE.json's hybrid configuration) only the new batches get
  // descriptors -- as a new segment -- instead of re-deriving all of them (11 us per batch: 3.3 ms per query at 300 batches).
  struct ScanSegment {
    const void* d_batches = nullptr; const int32_t* d_prefix = nullptr; int nbatches = 0; int total_chunks = 0; int needs_slow = 0;
    PathCounts paths;
    int64_t rows = 0, algo_bytes = 0, updated_cols = 0, deleted_batches = 0;
    size_t covered = 0;                          // batches of the store's snapshot this segment looked at (passing or skipped)
    std::vector<const StoredBatch*> batches;     // those that pass the stats check, in order
  };
  struct ScanCache {
    const sd_store* store = nullptr; int64_t version = -1; std::vector<int32_t> buckets; std::string lit_key;
    std::vector<ScanSegment> segs;
    std::vector<uint64_t> snap_uids;             // uid of every snapshot batch the segments cover, in order
    int64_t seen = 0, skipped = 0;
    int consolidations = 0;
    bool valid = false;
  } cache;
  Arena cache_arena;
  PinnedArena pinned;             // staging of descriptor uploads (valid until the next reset)
  // MODE_HASH group table + the launches of this execution (replayed after a grow)
  HashTable hash = {};
  uint32_t hash_capacity = 0;
  uint64_t* d_hash_ident = nullptr;
  bool hash_init = false;
  struct Launch { const void* d_batches; const int32_t* d_prefix; int nbatches; int total_chunks; int batch_base; int needs_slow; PathCounts paths; };
  // MODE_PROJECT output records + the batches of this execution (records carry a batch ordinal)
  uint8_t* d_out = nullptr;
  int64_t out_cap = 0;
  uint64_t* h_recs = nullptr;     // page-locked read-back staging of the projection records
  size_t h_recs_cap = 0;
  RowWriterBuffers roww;          // device row writer (sd_rows.cu): offsets, rows, string-source tables
  int64_t dev_rows_len = -1;      // >= 0: the finished rows of this execution are roww.d_rows[0, dev_rows_len) (not finished_rows)
  unsigned long long* d_out_count = nullptr;
  std::vector<const StoredBatch*> exec_batches;
  // the stores this execution may still read (hash-table string keys, MIN / MAX(STRING) slots and projected strings refer to
  // records in a store's memory): released once the result is materialised, by sd_plan_reset and sd_plan_destroy
  HeldPins pins;
  std::vector<uint8_t> finished_rows;   // rows of the last sd_plan_finish (re-served when the caller's buffer was too small)
  int64_t finished_nrows = -1;
  std::vector<Launch> launch_log;
  // grouping sets: the roll-up table of the fine groups into (keys, gid), and the plan's tables the roll-up kernel reads
  HashTable rollup = {};
  uint32_t rollup_capacity = 0;
  int32_t* d_rollup_meta = nullptr;
  size_t rollup_meta_cap = 0;
  double rollup_info[4] = {0, 0, 0, 0};   // sdx_plan_rollup_info
  cudaEvent_t ev_rollup[2] = {nullptr, nullptr};
  // what every kernel launch since the last reset ran (sdx_plan_launch_log): SDX_LAUNCH_WORDS words per launch
  std::vector<int64_t> launch_records;
  int replay_kind = SDX_REPLAY_NONE;   // why the launches being issued repeat earlier ones
  int64_t metrics[SD_NUM_METRICS] = {0};
  float agg_ms = 0;
  bool have_timing = false;
};

namespace {

std::string literal_key(const sd_plan* p) {
  std::string k;
  for (auto& l : p->lits) {
    k.append(reinterpret_cast<const char*>(&l.is_null), 4);
    k.append(reinterpret_cast<const char*>(&l.i), 8);
    k.append(reinterpret_cast<const char*>(&l.d), 8);
    if (l.s) k.append(l.s, (size_t)l.slen);
    k.push_back('|');
  }
  return k;
}

constexpr size_t STATE_HDR = 8;   // uint64 words in front of the running result: [0] rows scanned, [1] rows passed

int ensure_result(sd_plan* p, size_t entries) {
  if (entries > p->result_cap || !p->d_state) {
    SD_CUDA(cudaSetDevice(p->device));
    const size_t cap = std::max<size_t>(entries, 64);
    uint64_t* ns = nullptr;
    SD_CUDA(cudaMalloc(&ns, (STATE_HDR + cap) * 8));
    if (p->d_state) {   // the counters of the running execution move with the table
      SD_CUDA(cudaStreamSynchronize(p->stream));
      SD_CUDA(cudaMemcpy(ns, p->d_state, STATE_HDR * 8, cudaMemcpyDeviceToDevice));
      cudaFree(p->d_state);
    } else {
      SD_CUDA(cudaMemset(ns, 0, STATE_HDR * 8));
    }
    p->d_state = ns;
    p->d_result = ns + STATE_HDR;
    p->d_counters = reinterpret_cast<unsigned long long*>(ns);
    p->result_cap = cap;
    p->result_init = false;
  }
  if (STATE_HDR + p->result_cap > p->h_pinned_cap) {
    if (p->h_pinned) { SD_CUDA(cudaStreamSynchronize(p->stream)); cudaFreeHost(p->h_pinned); }
    p->h_pinned_cap = STATE_HDR + p->result_cap;
    SD_CUDA(cudaMallocHost(&p->h_pinned, p->h_pinned_cap * 8));
  }
  return 0;
}

// words of the running result for `ngroups` groups: [ngroups][slots], then the moment aggregates' K words [ngroups][shifts]
static size_t result_words(const PlanSpec& sp, int ngroups) { return (size_t)ngroups * (sp.slots.size() + sp.shifts.size()); }

// (re)initialise the running result with the slot identities (K words: SHIFT_EMPTY) for `ngroups` groups (async: the pinned
// staging buffer outlives the copy)
int init_result(sd_plan* p, int ngroups) {
  const int ns = (int)p->spec.slots.size();
  const size_t ne = (size_t)ngroups * ns, nw = result_words(p->spec, ngroups);
  int rc = ensure_result(p, nw);
  if (rc) return rc;
  SD_CUDA(cudaStreamSynchronize(p->stream));   // the staging buffer may still be in use by a previous read-back
  uint64_t* hid = p->h_pinned + STATE_HDR;
  for (size_t e = 0; e < ne; e++) {
    hid[e] = slot_initial(p->spec.slots[e % ns].op);
  }
  for (size_t e = ne; e < nw; e++) hid[e] = SHIFT_EMPTY;
  SD_CUDA(cudaMemcpyAsync(p->d_result, hid, nw * 8, cudaMemcpyHostToDevice, p->stream));
  p->result_init = true;
  return 0;
}

// group id of one key value in the query-global dictionary of key k
int key_id(sd_plan* p, int k, const std::string& s) {
  auto it = p->key_ids[k].find(s);
  if (it != p->key_ids[k].end()) return it->second;
  const int id = (int)p->key_vals[k].size();
  p->key_ids[k].emplace(s, id);
  p->key_vals[k].push_back(s);
  return id;
}
int key_null(sd_plan* p, int k) {
  if (p->key_null_id[k] < 0) {
    p->key_null_id[k] = (int)p->key_vals[k].size();
    p->key_vals[k].push_back(std::string());   // placeholder; identified by key_null_id
  }
  return p->key_null_id[k];
}

// when dictionaries grew between launches of one execution the dense group table is re-indexed
int remap_result(sd_plan* p, const int32_t* old_radix, int old_groups, const int32_t* new_radix, int new_groups) {
  const int ns = (int)p->spec.slots.size(), nk = (int)p->spec.keys.size(), nsh = (int)p->spec.shifts.size();
  std::vector<uint64_t> oldh(result_words(p->spec, old_groups));
  SD_CUDA(cudaStreamSynchronize(p->stream));
  SD_CUDA(cudaMemcpy(oldh.data(), p->d_result, oldh.size() * 8, cudaMemcpyDeviceToHost));
  int rc = init_result(p, new_groups);
  if (rc) return rc;
  SD_CUDA(cudaStreamSynchronize(p->stream));
  std::vector<uint64_t> newh(result_words(p->spec, new_groups));
  SD_CUDA(cudaMemcpy(newh.data(), p->d_result, newh.size() * 8, cudaMemcpyDeviceToHost));
  for (int g = 0; g < old_groups; g++) {
    int idx[MAX_KEYS], rem = g;
    for (int k = nk - 1; k >= 0; k--) { idx[k] = rem % old_radix[k]; rem /= old_radix[k]; }
    int ng = 0;
    for (int k = 0; k < nk; k++) ng = ng * new_radix[k] + idx[k];
    memcpy(&newh[(size_t)ng * ns], &oldh[(size_t)g * ns], (size_t)ns * 8);
    if (nsh) memcpy(&newh[(size_t)new_groups * ns + (size_t)ng * nsh], &oldh[(size_t)old_groups * ns + (size_t)g * nsh], (size_t)nsh * 8);
  }
  SD_CUDA(cudaMemcpy(p->d_result, newh.data(), newh.size() * 8, cudaMemcpyHostToDevice));
  return 0;
}

constexpr int REG_GROUPS_MAX = 8;
// local memory the two-CTA kernel of a dense group-by may use beyond its one-CTA kernel: Q1's spills 8 bytes (three local
// accesses in its SASS); plans whose per-row state does not fit 96 registers spill hundreds of bytes and stay at one CTA
constexpr size_t TWO_CTA_SPILL_SLACK = 16;
int resolve_kernel(const sd_plan_desc& desc, const CodegenOptions& opt, int device, KernelEntry* out, PlanSpec* spec_out);

struct BuiltScan {
  const void* d_batches = nullptr; const int32_t* d_prefix = nullptr; int nbatches = 0; int total_chunks = 0;
  int64_t rows = 0, algo_bytes = 0, updated_cols = 0, deleted_batches = 0;
  int needs_slow = 0;   // some batch needs the kernel variant with the per-row paths
  PathCounts paths;
  int needs_hash = 0;   // a key column of a dense-table plan is a raw (variable-width) string in some batch
};

// Build the device descriptors + per-batch tables for a list of resident batches.
// `up` is the stream the descriptors are uploaded on (from page-locked staging: the caller is never blocked); the
// scan must be ordered after it.
int build_scan(sd_plan* p, const std::vector<const StoredBatch*>& list, Arena& arena, cudaStream_t up, BuiltScan* out) {
  const PlanSpec& sp = p->spec;
  const int nc = (int)sp.cols.size();
  const size_t bstride = sizeof(DevBatch<1>) - sizeof(DevCol) + (size_t)std::max(nc, 1) * sizeof(DevCol);
  const int nt = (int)sp.tables.size();
  // SD_TUNE_NO_SCAN_IMAGES=1: the staged loads read the verbatim values (read per build, so one process can compare both)
  const char* no_img_env = getenv("SD_TUNE_NO_SCAN_IMAGES");
  const bool use_images = p->kernel.staged && !(no_img_env && atoi(no_img_env) > 0);
  std::vector<uint8_t> hb(bstride * std::max<size_t>(list.size(), 1), 0);
  std::vector<int32_t> prefix(list.size() + 1, 0);
  std::vector<uint8_t> aux;
  std::vector<size_t> aux_off(list.size(), 0);
  for (size_t bi = 0; bi < list.size(); bi++) {
    const StoredBatch& sb = *list[bi];
    uint8_t* rec = hb.data() + bi * bstride;
    DevBatch<1>* hdr = reinterpret_cast<DevBatch<1>*>(rec);
    hdr->num_rows = sb.num_rows;
    hdr->num_deletes = sb.num_deletes;
    hdr->deletes = sb.dev_deletes;
    bool all_fast = sb.dev_deletes == nullptr;
    bool base_fast = true;   // every base column can take the vector path (deltas / deletes aside)
    bool simple_enc = true;  // every column has a directly addressable encoding (NULLs allowed)
    bool any_delta = false;
    if (sb.dev_deletes) out->deleted_batches++;
    DevCol* dc = reinterpret_cast<DevCol*>(rec + (sizeof(DevBatch<1>) - sizeof(DevCol)));
    for (int c = 0; c < nc; c++) {
      const int t = sb.positional ? c : sp.cols[c].table_ordinal;
      if (t < 0 || t >= (int)sb.cols.size() || !sb.cols[t].present)
        return set_error(SD_ERR_INVALID, "batch %lld: table column %d is not resident", (long long)sb.batch_id, t);
      const StoredCol& sc = sb.cols[t];
      if (!sc.unsupported.empty()) return set_error(SD_ERR_UNSUPPORTED, "column %d: %s", t, sc.unsupported.c_str());
      dc[c] = sc.dev;
      {   // the scan image, when the kernel's decode of this column's kind reproduces the verbatim element from it
        const int k = sp.kinds[c];
        const bool match = sc.img_dict ? ((k == K_F64 && sc.img_ew == 8) || (k == K_F32 && sc.img_ew == 4))
                                       : ((k == K_I64 && sc.img_ew == 8) || (k == K_I32 && sc.img_ew == 4) || (k == K_I16 && sc.img_ew == 2) ||
                                          (k == K_CODE && ((sc.dev.enc == ENC_DICTIONARY && sc.img_ew == 2) || (sc.dev.enc == ENC_BIG_DICTIONARY && sc.img_ew == 4))));
        if (!(use_images && sc.dev.img && match && !sc.has_nulls)) { dc[c].img = nullptr; dc[c].img_tab = nullptr; dc[c].img_w = 0; dc[c].img_n = 0; }
      }
      all_fast = all_fast && sc.fast;
      {
        const bool simple = (sp.kinds[c] == K_CODE && (sc.dev.enc == ENC_DICTIONARY || sc.dev.enc == ENC_BIG_DICTIONARY || sc.dev.enc == ENC_STR_RAW)) ||
                            (sp.kinds[c] != K_CODE && sc.dev.enc == ENC_UNCOMPRESSED);
        simple_enc = simple_enc && simple && (!sc.has_nulls || sp.cols[c].nullable);   // NULLs in a column the plan calls non-nullable: per-row path
        any_delta = any_delta || sc.delta[0].present || sc.delta[1].present;
      }
      base_fast = base_fast && !sc.has_nulls && ((sp.kinds[c] == K_CODE && (sc.dev.enc == ENC_DICTIONARY || sc.dev.enc == ENC_BIG_DICTIONARY || sc.dev.enc == ENC_STR_RAW)) ||
                                                 (sp.kinds[c] != K_CODE && sc.dev.enc == ENC_UNCOMPRESSED));
      out->algo_bytes += sc.algo_bytes;
      if (sc.delta[0].present || sc.delta[1].present) out->updated_cols++;
      for (int d = 0; d < 2; d++) if (sc.delta[d].present) out->algo_bytes += sc.delta[d].len;
    }
    if (sb.dev_deletes) out->algo_bytes += 12 + 4 * (int64_t)sb.num_deletes;
    hdr->flags = all_fast ? BATCH_ALL_FAST : (base_fast ? BATCH_FAST_OVERLAY : ((simple_enc && !any_delta && !sb.dev_deletes) ? BATCH_FAST_NULLS : 0));
    if (!(hdr->flags == BATCH_ALL_FAST || (hdr->flags == BATCH_FAST_NULLS && p->kernel.staged))) out->needs_slow = 1;
    out->paths.n[hdr->flags == BATCH_ALL_FAST ? 0 : hdr->flags == BATCH_FAST_NULLS ? 1 : hdr->flags == BATCH_FAST_OVERLAY ? 2 : 3]++;
    for (int c = 0; c < nc; c++) {   // only the staged loads of the staged-only kernel variant read images (launch_scan)
      const int k = sp.kinds[c];
      const int64_t verbatim = k == K_CODE ? (dc[c].enc == ENC_DICTIONARY ? 2 : 4) : kind_stage_width(k);
      const int64_t narrow = hdr->flags && dc[c].img ? dc[c].img_w : verbatim;
      out->paths.streamed[0] += verbatim * sb.num_rows;
      out->paths.streamed[1] += narrow * sb.num_rows;
      if (hdr->flags) {
        PathCounts& pc = out->paths;
        pc.width[0][c] = (uint8_t)std::max<int64_t>(pc.width[0][c], verbatim);
        pc.width[1][c] = (uint8_t)std::max<int64_t>(pc.width[1][c], narrow);
        if (dc[c].img) pc.img_n[c] = std::max(pc.img_n[c], dc[c].img_n);
      }
    }
    // per-batch tables: [int32 offset x nt][pad 8][uint64 kpack x nt][tables]; every table is indexed by the
    // unified dictionary code; key maps of <= 8 codes are also packed one byte per code into kpack
    if (nt) {
      while (aux.size() % 16) aux.push_back(0);
      aux_off[bi] = aux.size();
      const size_t base = aux.size();
      const size_t kp_off = ((4 * (size_t)nt + 7) & ~size_t(7));
      aux.resize(base + kp_off + 8 * (size_t)nt, 0xff);
      for (int ti = 0; ti < nt; ti++) {
        const TableSpec& ts = sp.tables[ti];
        const StoredCol& sc = sb.cols[sb.positional ? ts.col : sp.cols[ts.col].table_ordinal];
        const int n = sc.dev.dict_n;                         // NULL code of a nullable column
        const bool nullable = sp.cols[ts.col].nullable != 0;
        if (sc.raw_str) {   // no code space: predicates / keys of this batch work on the bytes (the table stays empty)
          if (ts.kind == TABLE_KEYMAP) out->needs_hash = 1;   // a dense group table needs dictionary ids: this plan must use the hash table
          while (aux.size() % 8) aux.push_back(0);
          const int32_t off0 = (int32_t)(aux.size() - base);
          memcpy(aux.data() + base + 4 * (size_t)ti, &off0, 4);
          continue;
        }
        // codes: [0,n) base dictionary; n = NULL (nullable columns) or an unused placeholder when update
        // deltas appended strings; (n, ...) strings that occur only in update deltas
        const int ncodes = std::max((int)sc.dict_strings.size(), nullable ? n + 1 : n);
        while (aux.size() % 8) aux.push_back(0);
        const int32_t off = (int32_t)(aux.size() - base);
        memcpy(aux.data() + base + 4 * (size_t)ti, &off, 4);
        uint64_t kpack = ~0ull;
        bool packable = ts.kind == TABLE_KEYMAP && ncodes <= 8;
        uint8_t packed[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        if (ts.kind == TABLE_TRUTH) {
          for (int code = 0; code < ncodes; code++) {
            const bool isnull = code == n || code >= (int)sc.dict_strings.size();
            const std::string* s = isnull ? nullptr : &sc.dict_strings[code];
            aux.push_back((uint8_t)eval_string_predicate(sp, ts.node, s ? s->data() : nullptr, s ? (int)s->size() : 0, p->lits.data()));
          }
        } else if (ts.kind == TABLE_KEYPTR) {   // device address of every code's [len][bytes] record
          // FIRST / LAST of a STRING column return the winning row's own value: one that exists only in an update delta has no
          // device record to point at, so the plan is refused rather than answering NULL for it
          bool order_input = false;
          for (const auto& m : sp.agg_map)
            if (m.family == AGG_ORDER && m.hold == HOLD_REF && sp.exprs[sp.slots[(size_t)m.value_slot].node].a == ts.col) order_input = true;
          if (order_input && ts.key < 0)
            for (int code = n + 1; code < (int)sc.dict_strings.size(); code++)
              if (code >= (int)sc.dict_rec_ptr.size() || sc.dict_rec_ptr[code] == 0)
                return set_error(SD_ERR_UNSUPPORTED, "batch %lld: FIRST / LAST of a STRING column whose update deltas hold strings the "
                                 "batch's dictionary does not (compact the batch first)", (long long)sb.batch_id);
          for (int code = 0; code < ncodes; code++) {
            const int64_t ptr = code < (int)sc.dict_rec_ptr.size() ? sc.dict_rec_ptr[code] : 0;
            aux.insert(aux.end(), reinterpret_cast<const uint8_t*>(&ptr), reinterpret_cast<const uint8_t*>(&ptr) + 8);
          }
        } else {
          for (int code = 0; code < ncodes; code++) {
            const bool isnull = code == n || code >= (int)sc.dict_strings.size();
            const int32_t id = isnull ? (nullable ? key_null(p, ts.key) : 0) : key_id(p, ts.key, sc.dict_strings[code]);
            aux.insert(aux.end(), reinterpret_cast<const uint8_t*>(&id), reinterpret_cast<const uint8_t*>(&id) + 4);
            if (packable) { if (id >= 255) packable = false; else packed[code] = (uint8_t)id; }
          }
          if (packable) memcpy(&kpack, packed, 8);
        }
        memcpy(aux.data() + base + kp_off + 8 * (size_t)ti, &kpack, 8);
      }
    }
    out->rows += sb.num_rows;
    prefix[bi + 1] = prefix[bi] + (sb.num_rows + p->chunk_rows - 1) / p->chunk_rows;
  }
  // NULL key ids are only materialised when a nullable key column is present in the plan
  uint8_t* d_aux = nullptr;
  if (!aux.empty()) {
    d_aux = arena.alloc(aux.size() + 16, 16);
    uint8_t* h_aux = p->pinned.alloc(aux.size());
    if (!d_aux || !h_aux) return SD_ERR_CUDA;
    memcpy(h_aux, aux.data(), aux.size());
    SD_CUDA(cudaMemcpyAsync(d_aux, h_aux, aux.size(), cudaMemcpyHostToDevice, up));
    for (size_t bi = 0; bi < list.size(); bi++) reinterpret_cast<DevBatch<1>*>(hb.data() + bi * bstride)->aux = d_aux + aux_off[bi];
  }
  uint8_t* d_b = arena.alloc(hb.size() + 16, 16);
  uint8_t* d_p = arena.alloc(prefix.size() * 4 + 16, 16);
  uint8_t* h_b = p->pinned.alloc(hb.size());
  uint8_t* h_p = p->pinned.alloc(prefix.size() * 4);
  if (!d_b || !d_p || !h_b || !h_p) return SD_ERR_CUDA;
  memcpy(h_b, hb.data(), hb.size());
  memcpy(h_p, prefix.data(), prefix.size() * 4);
  SD_CUDA(cudaMemcpyAsync(d_b, h_b, hb.size(), cudaMemcpyHostToDevice, up));
  SD_CUDA(cudaMemcpyAsync(d_p, h_p, prefix.size() * 4, cudaMemcpyHostToDevice, up));
  out->d_batches = d_b;
  out->d_prefix = reinterpret_cast<const int32_t*>(d_p);
  out->nbatches = (int)list.size();
  out->total_chunks = prefix.back();
  return 0;
}

void table_free(HashTable& t) {
  if (t.state) cudaFree(t.state);
  if (t.keys) cudaFree(t.keys);
  if (t.knull) cudaFree(t.knull);
  if (t.vals) cudaFree(t.vals);
  if (t.shifts) cudaFree(t.shifts);
  if (t.overflow) cudaFree(t.overflow);
  t = HashTable{};
}
// device memory of a hash group table of `capacity` entries (state not initialised)
int table_alloc(HashTable& t, uint32_t capacity, int nk, int ns, int nsh) {
  table_free(t);
  SD_CUDA(cudaMalloc(&t.state, (size_t)capacity * 4));
  SD_CUDA(cudaMalloc(&t.keys, (size_t)capacity * nk * 8));
  SD_CUDA(cudaMalloc(&t.knull, (size_t)capacity * 4));
  SD_CUDA(cudaMalloc(&t.vals, (size_t)capacity * ns * 8));
  if (nsh) SD_CUDA(cudaMalloc(&t.shifts, (size_t)capacity * nsh * 8));
  SD_CUDA(cudaMalloc(&t.overflow, 1024));   // [0] overflow flag, [8] key count; the rest: diagnostic histograms (SD_EXP_VERIFY builds)
  SD_CUDA(cudaMemset(t.overflow, 0, 1024));
  t.count = t.overflow + 8;
  t.mask = capacity - 1;
  t.max_probe = std::min<uint32_t>(capacity, 4096);
  return 0;
}
void hash_free(sd_plan* p) {
  table_free(p->hash);
  p->hash_capacity = 0;
}

int hash_ident(sd_plan* p);
int hash_ensure(sd_plan* p, uint32_t capacity) {
  const int ns = (int)p->spec.slots.size(), nk = std::max<int>(1, (int)p->spec.keys.size());
  if (p->hash_capacity != capacity) {
    p->hash_capacity = 0;
    int rc = table_alloc(p->hash, capacity, nk, ns, (int)p->spec.shifts.size());
    if (rc) return rc;
    p->hash_capacity = capacity;
    p->hash_init = false;
  }
  int rc = hash_ident(p);
  if (rc) return rc;
  if (!p->hash_init) {
    rc = hash_table_init(p->stream, p->hash, capacity, ns, p->d_hash_ident, (int)p->spec.shifts.size());
    if (rc) return rc;
    p->hash_init = true;
  }
  return 0;
}

// the slot identities a hash group table starts from (device copy, made once)
int hash_ident(sd_plan* p) {
  const int ns = (int)p->spec.slots.size();
  if (!p->d_hash_ident) {
    std::vector<uint64_t> id(ns);
    for (int s = 0; s < ns; s++) id[s] = slot_initial(p->spec.slots[s].op);
    SD_CUDA(cudaMalloc(&p->d_hash_ident, (size_t)std::max(ns, 1) * 8));
    SD_CUDA(cudaMemcpy(p->d_hash_ident, id.data(), (size_t)ns * 8, cudaMemcpyHostToDevice));
  }
  return 0;
}

int ensure_out(sd_plan* p, int64_t cap_records) {
  const int64_t rec = (p->spec.mode == MODE_MUTATE ? 16 : 8) + 8 * (int64_t)std::max<size_t>(p->spec.proj.size(), 1);
  if (!p->d_out_count) { SD_CUDA(cudaMalloc(&p->d_out_count, 64)); SD_CUDA(cudaMemset(p->d_out_count, 0, 64)); }
  if (cap_records > p->out_cap) {
    if (p->d_out) cudaFree(p->d_out);
    p->d_out = nullptr;
    SD_CUDA(cudaMalloc(&p->d_out, (size_t)(cap_records * rec)));
    p->out_cap = cap_records;
  }
  return 0;
}

// device time of this execution's launches (sum over the per-launch event pairs; the span as a fallback)
static void update_agg_time(sd_plan* p) {
  if (!p->have_timing) return;
  float total = 0;
  bool ok = p->ev_used > 0 && p->ev_used == (size_t)p->metrics[7];
  for (size_t i = 0; ok && i < p->ev_used; i++) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, p->ev_pairs[i].first, p->ev_pairs[i].second) != cudaSuccess) { ok = false; break; }
    total += ms;
  }
  if (!ok) { float ms = 0; if (cudaEventElapsedTime(&ms, p->ev_start, p->ev_stop) == cudaSuccess) total = ms; else return; }
  p->agg_ms = total;
}

// the kernel variant of the plan for this execution / launch
int plan_variant(sd_plan* p, int litnull, int slow, const KernelEntry** out) {
  const int idx = (litnull ? 1 : 0) | (slow ? 2 : 0);
  if (idx == 0) { *out = &p->kernel; return 0; }
  if (!p->variant_state[idx]) {
    CodegenOptions opt;
    opt.lit_nullable = litnull ? 1 : 0;
    opt.slow_paths = slow ? 1 : 0;
    opt.force_hash = p->force_hash ? 1 : 0;
    sd_plan_desc dv = p->spec.desc_view();
    int rc = resolve_kernel(dv, opt, p->device, &p->variant[idx], nullptr);
    if (rc) return rc;
    p->variant_state[idx] = 1;
  }
  *out = &p->variant[idx];
  return 0;
}

int launch_scan(sd_plan* p, const void* d_batches, const int32_t* d_prefix, int nbatches, int total_chunks, int needs_slow,
                const PathCounts& paths, const std::vector<const StoredBatch*>* blist = nullptr, int replay_batch_base = -1);

// A dense-table plan (dictionary-string keys) has to give up its table: too many key combinations, or a key column
// arrives as raw variable-width strings (no dictionary ids).  The plan becomes its hash-table variant for good and
// whatever this execution has launched so far is rebuilt (the per-batch tables differ) and launched again.
int switch_to_hash(sd_plan* p) {
  CodegenOptions opt;
  opt.force_hash = 1;
  PlanSpec hspec;
  KernelEntry hk;
  sd_plan_desc dv = p->spec.desc_view();
  int rc = resolve_kernel(dv, opt, p->device, &hk, &hspec);
  if (rc) return rc;
  const std::vector<sd_plan::Launch> earlier(p->launch_log);
  const std::vector<const StoredBatch*> exec(p->exec_batches);
  p->launch_log.clear();
  p->exec_batches.clear();
  p->spec = hspec;
  p->kernel = hk;
  p->force_hash = true;
  for (int v = 0; v < 4; v++) p->variant_state[v] = 0;
  p->active = nullptr;
  p->last_kernel = nullptr;
  p->last_smem = (size_t)-1;
  p->result_init = false;
  p->hash_init = false;
  p->cache.valid = false;
  p->chunk_rows = CHUNK_ROWS;
  SD_CUDA(cudaMemsetAsync(p->d_counters, 0, 64, p->stream));
  p->replay_kind = SDX_REPLAY_HASH_SWITCH;
  for (auto& l : earlier) {
    std::vector<const StoredBatch*> list(exec.begin() + l.batch_base, exec.begin() + l.batch_base + l.nbatches);
    BuiltScan bs;
    rc = build_scan(p, list, p->scratch, p->stream, &bs);
    if (rc) return rc;
    rc = launch_scan(p, bs.d_batches, bs.d_prefix, bs.nbatches, bs.total_chunks, bs.needs_slow, bs.paths, &list);
    if (rc) return rc;
  }
  p->replay_kind = SDX_REPLAY_NONE;
  return 0;
}

// a dense group table holds at most this many key combinations; beyond it the plan becomes its hash-table variant
constexpr int64_t DENSE_GROUPS_MAX = 1 << 16;
// key combinations of the dense table with the dictionaries seen so far
int64_t dense_groups(const sd_plan* p) {
  int64_t ng = 1;
  for (size_t k = 0; k < p->spec.keys.size(); k++) ng *= std::max<int64_t>(1, (int64_t)p->key_vals[k].size());
  return ng;
}

int launch_scan(sd_plan* p, const void* d_batches, const int32_t* d_prefix, int nbatches, int total_chunks, int needs_slow,
                const PathCounts& paths, const std::vector<const StoredBatch*>* blist, int replay_batch_base) {
  const bool replay = replay_batch_base >= 0;
  if (!replay && p->spec.mode == MODE_GROUPS) {   // dense table still possible with the dictionaries seen so far?
    if (dense_groups(p) > DENSE_GROUPS_MAX) {
      if (!blist) return set_error(SD_ERR_STATE, "dense group table overflow without a batch list");
      int rc = switch_to_hash(p);
      if (rc) return rc;
      BuiltScan bs;
      rc = build_scan(p, *blist, p->scratch, p->stream, &bs);
      if (rc) return rc;
      return launch_scan(p, bs.d_batches, bs.d_prefix, bs.nbatches, bs.total_chunks, bs.needs_slow, bs.paths, blist);
    }
  }
  int batch_base = replay ? replay_batch_base : (int)p->exec_batches.size();
  if (!replay && p->spec.mode != MODE_NOKEY) {
    p->launch_log.push_back({d_batches, d_prefix, nbatches, total_chunks, batch_base, needs_slow, paths});
    if (blist) p->exec_batches.insert(p->exec_batches.end(), blist->begin(), blist->end());
  } else if (!replay && p->spec.norder > 0 && blist) {   // no keys: only the batch sequence of FIRST / LAST's order keys
    p->exec_batches.insert(p->exec_batches.end(), blist->begin(), blist->end());
  }
  p->finished_nrows = -1;
  p->dev_rows_len = -1;
  if (nbatches == 0 || total_chunks == 0) return 0;
  const PlanSpec& sp = p->spec;
  const int ns = (int)sp.slots.size(), nk = (int)sp.keys.size();
  // group radices from the current key dictionaries
  int32_t radix[MAX_KEYS] = {1, 1, 1, 1};
  int ngroups = 1;
  for (int k = 0; k < nk && sp.mode == MODE_GROUPS; k++) {
    radix[k] = std::max<int>(1, (int)p->key_vals[k].size());
    ngroups *= radix[k];
  }
  const size_t ne = (size_t)ngroups * ns;
  // Where the dense group table lives (decided per launch from its size):
  //   registers (kernel variant, <= 8 groups) > per-thread private shared-memory copies > one shared-memory copy
  //   per CTA with atomics > global atomics on the running result.
  // What is left of the SM's shared memory (per target CTA) becomes the ring of the staged fast path.
  const KernelEntry* k = &p->kernel;
  {   // a NULL literal needs the variant whose generated code carries literal null flags; batches with deltas, deletes
      // or encodings that are not directly addressable need the variant that carries the per-row paths
    bool any_null = false;
    for (auto& l : p->lits) any_null = any_null || l.is_null;
    static const bool force_full = getenv("SD_TUNE_FULL_KERNEL") != nullptr;   // measurement aid
    int rc = plan_variant(p, any_null, needs_slow || force_full, &k);
    if (rc) return rc;
  }
  int table_mode = TABLE_PRIVATE;
  int fresh = 0;
  const int nshift = (int)sp.shifts.size();
  if (sp.mode == MODE_GROUPS && ngroups <= REG_GROUPS_MAX && k == &p->kernel && p->kernel.staged && getenv("SD_TUNE_REG_GROUPS") && nshift == 0) {
    // experimental (opt-in): measured slower than the private shared-memory tables, see DESIGN.md
    if (p->kernel_reg_state == 0) {
      CodegenOptions opt;
      opt.reg_groups = REG_GROUPS_MAX;
      sd_plan_desc dv = sp.desc_view();
      p->kernel_reg_state = resolve_kernel(dv, opt, p->device, &p->kernel_reg, nullptr) == 0 ? 1 : -1;
    }
    // the accumulators are reduced through the ring, which keeps the verbatim layout below and at least two stages
    if (p->kernel_reg_state == 1 && 2 * p->kernel_reg.stage_bytes >= ne * THREADS * 8) {
      k = &p->kernel_reg;
      table_mode = TABLE_REGS;
    }
  }
  // Two CTAs per SM for dense group-bys.  With images the per-row work, not the ring, bounds the kernel, and a second CTA
  // doubles the consumer warps that hide its latency.  The staged-only variant has a kernel built for two CTAs
  // (scan_aggregate_kernel_2cta, <= 96 registers) that reads the ring layout from the launch (RingArgs): each column's
  // stage region sized by the widest element a batch of the launch streams (its scan image, or its verbatim width with
  // dictionary codes at 2 or 4 bytes), each image table by the most entries a batch has.  A launch takes it when that
  // kernel spills at most TWO_CTA_SPILL_SLACK bytes more than the one-CTA kernel, the tile state, the private table, the image tables and two compact
  // stages fit half the SM, and the occupancy query agrees; otherwise it runs as before the two-CTA kernel existed: the
  // plan's kernel, verbatim layout, one CTA.  SD_TUNE_RING_LAYOUT=verbatim or SD_TUNE_GROUP_CTAS=1 force the latter.
  const char* layout_env = getenv("SD_TUNE_RING_LAYOUT");
  const char* ctas_env = getenv("SD_TUNE_GROUP_CTAS");
  const bool slow_variant = k == &p->variant[2] || k == &p->variant[3];
  bool two_cta = sp.mode == MODE_GROUPS && table_mode != TABLE_REGS && (k->func2 || k->drv_func2) &&
                 !(layout_env && !strcmp(layout_env, "verbatim")) && !(ctas_env && atoi(ctas_env) == 1);
  if (two_cta) {
    size_t local1 = 0, local2 = 0;
    int rc = kernel_local_bytes(*k, false, &local1);
    if (!rc) rc = kernel_local_bytes(*k, true, &local2);
    if (rc) return rc;
    two_cta = local2 <= local1 + TWO_CTA_SPILL_SLACK;
  }
  const bool want_img = k->staged && !slow_variant && paths.streamed[1] < paths.streamed[0];
  const int nc = (int)sp.kinds.size();
  RingArgs ring;
  memset(&ring, 0, sizeof(ring));
  const size_t tile_smem = k->tile_smem;
  const size_t ring_fixed = 2 * MAX_STAGES * 8 + RING_ALIGN_SLACK;   // mbarriers + alignment of the ring
  size_t table_bytes, stage_bytes, ring_off, smem;
  int target_ctas, shift_cache_off, img_off, nstages;
  bool compact;
  for (int attempt = two_cta ? 2 : 1;; attempt = 1) {
    compact = attempt == 2;
    // stage and image-table layout: compact (RingArgs) or verbatim (the kernel's constants)
    stage_bytes = 0;
    size_t img_bytes = 0;
    for (int c = 0; c < nc; c++) {
      ring.stage_off[c] = (int32_t)stage_bytes;
      ring.img_col[c] = (int32_t)(img_bytes / 8);
      // + 128: a column with NULLs is copied from the 16-byte boundary below its first value of the tile, and every region
      // stays 128-byte aligned for the bulk copies
      stage_bytes += (size_t)k->tile_rows * (compact ? paths.width[want_img ? 1 : 0][c] : kind_stage_width(sp.kinds[c])) + 128;
      img_bytes += 8 * (size_t)(compact ? paths.img_n[c] : img_smem_words(sp.kinds[c]));
    }
    ring.stage_bytes = (int32_t)stage_bytes;
    target_ctas = table_mode == TABLE_REGS ? 1 : compact ? 2 : std::max(1, sp.min_ctas);
    const size_t min_ring = k->staged ? ring_fixed + 2 * stage_bytes + 128 : 0;
    table_bytes = (size_t)std::max(ns, 1) * (THREADS / 32) * 8;
    shift_cache_off = -1;
    auto img_fits = [&](size_t table, size_t budget) {   // the image tables sit between the group table and the ring
      return ((((tile_smem + table + 15) & ~size_t(15)) + img_bytes + 127) & ~size_t(127)) + min_ring <= budget;
    };
    if (sp.mode == MODE_GROUPS && table_mode != TABLE_REGS) {
      // moment aggregates: the shared-memory tables come with the CTA's copy of the K words behind them
      const size_t kc = (size_t)ngroups * nshift * 8;
      const size_t priv = ne * THREADS * 8 + kc, shared = ne * 8 + kc;
      // private copies are worth giving up CTAs per SM for; atomics are the last resort
      while (target_ctas > 1 && tile_smem + priv + min_ring > (size_t)p->smem_optin / target_ctas - 1024) target_ctas--;
      const size_t budget1 = (size_t)p->smem_optin / target_ctas - (target_ctas > 1 ? 1024 : 0);
      if (tile_smem + priv + min_ring <= budget1) { table_mode = TABLE_PRIVATE; table_bytes = priv; }
      else if (shared <= 64 * 1024 && tile_smem + shared + min_ring <= budget1) { table_mode = TABLE_SHARED_ATOMIC; table_bytes = shared; }
      else { table_mode = TABLE_GLOBAL_ATOMIC; table_bytes = 64; }
      if (nshift > 0 && table_mode != TABLE_GLOBAL_ATOMIC) shift_cache_off = (int)(tile_smem + table_bytes - kc);
    }
    const size_t budget = (size_t)p->smem_optin / target_ctas - (target_ctas > 1 ? 1024 : 0);
    if (compact && (target_ctas != 2 || table_mode != TABLE_PRIVATE || (want_img && !img_fits(table_bytes, budget)))) continue;
    // the per-chunk copies of the image tables, when the batches have images, the kernel is the staged-only variant (the one
    // with the per-row paths reads verbatim values) and the ring keeps at least two stages
    img_off = -1;
    size_t img_end = tile_smem + table_bytes;
    if (want_img && img_fits(table_bytes, budget)) {
      img_off = (int)((tile_smem + table_bytes + 15) & ~size_t(15));
      img_end = img_off + img_bytes;
    }
    ring_off = (img_end + 127) & ~size_t(127);
    nstages = 0;
    smem = ring_off;
    if (k->staged) {
      if (ring_off + min_ring > (size_t)p->smem_optin) return set_error(SD_ERR_UNSUPPORTED, "plan does not fit the shared-memory ring (%zu bytes per stage)", stage_bytes);
      const size_t avail = std::max(budget, ring_off + min_ring) - ring_off - ring_fixed;
      nstages = (int)std::min<size_t>(MAX_STAGES, avail / stage_bytes);
      if (const char* e = getenv("SD_TUNE_NSTAGES")) { int v = atoi(e); if (v >= 2 && v <= nstages) nstages = v; }
      smem = ring_off + ring_fixed + (size_t)nstages * stage_bytes;
    }
    if (smem != p->last_smem || k != p->last_kernel || compact != p->last_two_cta) {
      int occ = 0;
      int rc = kernel_prepare(*k, compact, smem, &occ);
      if (rc) return rc;
      if (occ < 1) return set_error(SD_ERR_CUDA, "kernel does not fit on an SM (smem %zu)", smem);
      p->max_ctas_per_sm = occ;
      p->last_smem = smem;
      p->last_kernel = k;
      p->last_two_cta = compact;
    }
    if (!compact || p->max_ctas_per_sm >= 2) break;
  }
  if (p->active != k) { p->active = k; p->kernel_name = k->origin + ":" + k->name + (table_mode == TABLE_REGS ? "+regtable" : ""); }
  if (sp.mode == MODE_HASH) {
    int rc = hash_ensure(p, p->hash_capacity ? p->hash_capacity : (1u << 16));
    if (rc) return rc;
  } else if (sp.mode == MODE_PROJECT || sp.mode == MODE_MUTATE) {
    int rc = ensure_out(p, p->out_cap ? p->out_cap : (int64_t(1) << 20));
    if (rc) return rc;
  } else if (!p->result_init) {
    if (table_mode == TABLE_GLOBAL_ATOMIC) {   // the kernel adds into the running result: it must hold the identities
      int rc = init_result(p, ngroups);
      if (rc) return rc;
    } else {                                     // the last CTA overwrites it (ScanArgs.fresh): nothing to upload
      int rc = ensure_result(p, result_words(sp, ngroups));
      if (rc) return rc;
      // the K words of moment aggregates behind it are claimed, not overwritten: SHIFT_EMPTY (all ones) before the first launch
      if (nshift) SD_CUDA(cudaMemsetAsync(p->d_result + ne, 0xff, (size_t)ngroups * nshift * 8, p->stream));
      fresh = 1;
      p->result_init = true;
    }
  } else if (ngroups != p->ngroups || memcmp(radix, p->radix, sizeof(radix)) != 0) {
    int rc = remap_result(p, p->radix, p->ngroups, radix, ngroups);
    if (rc) return rc;
  }
  p->ngroups = ngroups;
  memcpy(p->radix, radix, sizeof(radix));

  const int occ = p->max_ctas_per_sm;
  const int grid = std::min(total_chunks, p->num_sms * occ);
  if (table_mode != TABLE_GLOBAL_ATOMIC && (size_t)grid * ne > p->partials_cap) {
    if (p->d_partials) cudaFree(p->d_partials);
    p->partials_cap = (size_t)grid * ne * 2;
    SD_CUDA(cudaMalloc(&p->d_partials, p->partials_cap * 8));
  }
  ScanArgs args;
  memset(&args, 0, sizeof(args));
  args.batches = d_batches;
  args.chunk_prefix = d_prefix;
  args.nbatches = nbatches;
  args.total_chunks = total_chunks;
  args.partials = p->d_partials;
  args.result = p->d_result;
  args.shifts = nshift ? p->d_result + ne : nullptr;
  args.ticket = p->d_ticket;
  args.counters = p->d_counters;
  args.ngroups = ngroups;
  args.table_mode = table_mode;
  args.ring_off = (int32_t)ring_off;
  args.nstages = nstages;
  args.hash = p->hash;
  args.out_rows = p->d_out;
  args.out_count = p->d_out_count;
  args.out_cap = p->out_cap;
  args.batch_base = batch_base;
  args.chunk_rows = p->chunk_rows;
  args.fresh = fresh;
  args.shift_cache_off = shift_cache_off;
  args.img_off = img_off;
  memcpy(args.radix, radix, sizeof(radix));
  if (p->litpool_dirty) {   // STRING literal bytes -> device (once per set of literal values)
    std::vector<uint8_t> pool;
    p->lit_packed.assign(p->lits.size(), 0);
    for (size_t i = 0; i < p->lits.size(); i++) {
      if (p->spec.lit_wide[i]) {   // wide DECIMAL: the 128-bit value, little-endian, 16-byte aligned (sd::dec_lit)
        pool.resize((pool.size() + 15) & ~size_t(15), 0);
        p->lit_packed[i] = (int64_t)(((uint64_t)pool.size() << 32) | 16u);
        const i128 v = p->lits[i].is_null ? 0 : dec_from_bytes(reinterpret_cast<const uint8_t*>(p->lits[i].s), (size_t)p->lits[i].slen);
        pool.insert(pool.end(), reinterpret_cast<const uint8_t*>(&v), reinterpret_cast<const uint8_t*>(&v) + 16);
        continue;
      }
      if (p->lits[i].type != SD_STRING) continue;
      p->lit_packed[i] = (int64_t)(((uint64_t)pool.size() << 32) | (uint32_t)p->lits[i].slen);
      pool.insert(pool.end(), p->lits[i].s, p->lits[i].s + p->lits[i].slen);
    }
    if (!pool.empty()) {
      if (pool.size() > p->litpool_cap) {
        if (p->d_litpool) cudaFree(p->d_litpool);
        p->litpool_cap = pool.size() * 2 + 256;
        SD_CUDA(cudaMalloc(&p->d_litpool, p->litpool_cap));
      }
      uint8_t* h = p->pinned.alloc(pool.size());
      if (!h) return SD_ERR_CUDA;
      memcpy(h, pool.data(), pool.size());
      SD_CUDA(cudaMemcpyAsync(p->d_litpool, h, pool.size(), cudaMemcpyHostToDevice, p->stream));
    }
    p->litpool_dirty = false;
  }
  args.lit_pool = p->d_litpool;
  for (size_t i = 0; i < p->lits.size(); i++) {
    args.lits.i[i] = p->lits[i].type == SD_STRING || p->spec.lit_wide[i] ? p->lit_packed[i] : p->lits[i].i;
    args.lits.d[i] = p->lits[i].d;
    if (p->lits[i].is_null) args.lits.nullmask |= 1ull << i;
  }
  void* kargs[] = {&args, &ring};
  if (p->ev_used == p->ev_pairs.size() && p->ev_pairs.size() < 4096) {
    cudaEvent_t a = nullptr, b = nullptr;
    SD_CUDA(cudaEventCreate(&a));
    SD_CUDA(cudaEventCreate(&b));
    p->ev_pairs.emplace_back(a, b);
  }
  const bool own_pair = p->ev_used < p->ev_pairs.size();
  if (own_pair) SD_CUDA(cudaEventRecord(p->ev_pairs[p->ev_used].first, p->stream));
  if (!p->have_timing) SD_CUDA(cudaEventRecord(p->ev_start, p->stream));
  { int rc = kernel_launch(*k, compact, grid, smem, p->stream, kargs); if (rc) return rc; }
  if (p->launch_records.size() < (size_t)SDX_LAUNCH_LOG_MAX * SDX_LAUNCH_WORDS) {
    const int acc = sp.mode == MODE_NOKEY ? SDX_ACC_NOKEY : sp.mode == MODE_HASH ? SDX_ACC_HASH
                  : (sp.mode == MODE_PROJECT || sp.mode == MODE_MUTATE) ? SDX_ACC_ROWS
                  : table_mode == TABLE_PRIVATE ? SDX_ACC_PRIVATE : table_mode == TABLE_SHARED_ATOMIC ? SDX_ACC_SHARED_ATOMIC
                  : table_mode == TABLE_GLOBAL_ATOMIC ? SDX_ACC_GLOBAL_ATOMIC : SDX_ACC_REGTABLE;
    const int64_t rec[SDX_LAUNCH_WORDS] = {acc, k == &p->variant[2] || k == &p->variant[3], k == &p->variant[1] || k == &p->variant[3],
                                           nstages, k->tile_rows, p->chunk_rows, grid, ngroups, paths.n[0], paths.n[1], paths.n[2],
                                           paths.n[3], p->replay_kind, nbatches, total_chunks, paths.streamed[img_off >= 0 ? 1 : 0]};
    p->launch_records.insert(p->launch_records.end(), rec, rec + SDX_LAUNCH_WORDS);
  }
  SD_CUDA(cudaEventRecord(p->ev_stop, p->stream));
  if (own_pair) { SD_CUDA(cudaEventRecord(p->ev_pairs[p->ev_used].second, p->stream)); p->ev_used++; }
  p->have_timing = true;
  p->metrics[7]++;
  return 0;
}

int flush_pending(sd_plan* p) {
  if (p->pending.empty()) return 0;
  if (p->priv) {   // queue the expansion of compressed buffers first: it runs while the descriptors are being built
    int rc0 = store_flush_lz4(p->priv);
    if (rc0) return rc0;
  }
  std::vector<const StoredBatch*> list;
  for (auto& x : p->pending) list.push_back(x.sb);
  BuiltScan bs;
  // nothing below blocks the submitting thread: descriptors go out on the copy stream from page-locked staging, and
  // the scan is ordered after the copies and the expansions with events
  int rc = build_scan(p, list, p->scratch, p->priv ? p->priv->copy_stream : p->stream, &bs);
  if (rc) return rc;
  if (bs.needs_hash && p->spec.mode == MODE_GROUPS) {   // a key column came as raw strings: dense ids do not exist for it
    rc = switch_to_hash(p);
    if (rc) return rc;
    bs = BuiltScan();
    rc = build_scan(p, list, p->scratch, p->priv ? p->priv->copy_stream : p->stream, &bs);
    if (rc) return rc;
  }
  if (p->priv) {
    if (!p->priv->copies_done) SD_CUDA(cudaEventCreateWithFlags(&p->priv->copies_done, cudaEventDisableTiming));
    SD_CUDA(cudaEventRecord(p->priv->copies_done, p->priv->copy_stream));
    SD_CUDA(cudaStreamWaitEvent(p->stream, p->priv->copies_done, 0));
    for (int k = 0; k + 1 < p->priv->num_copy_streams; k++) {
      SD_CUDA(cudaEventRecord(p->priv->extra_done[k], p->priv->extra_streams[k]));
      SD_CUDA(cudaStreamWaitEvent(p->stream, p->priv->extra_done[k], 0));
    }
    rc = store_lz4_order(p->priv, p->stream);   // the scan reads what the expansions write
    if (rc) return rc;
  }
  p->metrics[3] += bs.updated_cols;
  p->metrics[4] += bs.deleted_batches;
  p->metrics[9] += bs.algo_bytes;
  rc = launch_scan(p, bs.d_batches, bs.d_prefix, bs.nbatches, bs.total_chunks, bs.needs_slow, bs.paths, &list);
  p->pending.clear();
  p->pending_bytes = 0;
  return rc;
}

bool batch_passes_stats(const sd_plan* p, const StoredBatch& sb) {
  if (p->spec.filter < 0 || sb.stats.empty()) return true;
  StatEval ev{p->spec, p->lits, sb.stats.data(), (int64_t)sb.stats.size(), 1 + 3 * sb.stats_ncols, sb.num_rows};
  Tri r;
  if (!ev.eval(p->spec.filter, &r)) return true;
  return r.isnull || r.v;   // only a definite FALSE skips the batch (:948-957)
}

// test hook (host only, no CUDA call): the batch-skipping decision of a plan for one stats row
int stats_pass_hook(const sd_plan_desc* desc, const sd_literal* lits, int32_t nlits, const void* stats, int64_t stats_len,
                    int32_t stats_ncols, int32_t num_rows, int32_t* pass) {
  if (!desc || !pass || (nlits > 0 && !lits)) return set_error(SD_ERR_INVALID, "sdx_stats_pass: null argument");
  PlanSpec spec;
  std::string err;
  int rc = analyze_plan(desc, spec, err);
  if (rc) return set_error(rc, "sdx_stats_pass: %s", err.c_str());
  if (nlits != (int)spec.literal_types.size()) return set_error(SD_ERR_INVALID, "sdx_stats_pass: plan has %zu literal slots", spec.literal_types.size());
  std::vector<sd_literal> lv(lits, lits + nlits);
  *pass = 1;
  if (spec.filter < 0 || !stats || stats_len <= 0) return 0;
  StatEval ev{spec, lv, reinterpret_cast<const uint8_t*>(stats), stats_len, 1 + 3 * stats_ncols, num_rows};
  Tri r;
  if (ev.eval(spec.filter, &r)) *pass = (r.isnull || r.v) ? 1 : 0;
  return 0;
}

// find the kernel for a codegen variant of the plan: ahead-of-time registry first, else NVRTC
int resolve_kernel(const sd_plan_desc& desc, const CodegenOptions& opt, int device, KernelEntry* out, PlanSpec* spec_out) {
  PlanSpec spec;
  std::string err;
  int rc = analyze_plan(&desc, spec, err, &opt);
  if (rc) return set_error(rc, "%s", err.c_str());
  static std::mutex registry_mutex;   // plans are created concurrently from many task threads
  std::lock_guard<std::mutex> lock(registry_mutex);
  for (auto& k : kernel_registry()) if (k.signature == spec.signature) { *out = k; out->tile_rows = THREADS * spec.rpt; if (spec_out) *spec_out = spec; return 0; }
  KernelEntry k;
  rc = jit_compile(spec, device, k);
  if (rc) return rc;
  kernel_registry().push_back(k);
  *out = k;
  out->tile_rows = THREADS * spec.rpt;
  if (spec_out) *spec_out = spec;
  return 0;
}

// HOLD_REF values: slots hold device addresses of [len][bytes] records -> their bytes, for every group at once
int fetch_agg_strings(sd_plan* p, const uint64_t* slots, size_t ngroups, StrMap& out) {
  const PlanSpec& sp = p->spec;
  const size_t ns = sp.slots.size();
  std::vector<int64_t> ptrs;
  for (auto& m : sp.agg_map) {
    if (m.hold != HOLD_REF) continue;
    for (size_t g = 0; g < ngroups; g++) { const uint64_t a = slots[g * ns + m.value_slot]; if (a && !out.count(a)) { out.emplace(a, std::string()); ptrs.push_back((int64_t)a); } }
  }
  if (ptrs.empty()) return 0;
  int64_t* d_ptrs = nullptr;
  SD_CUDA(cudaMalloc(&d_ptrs, ptrs.size() * 8));
  std::vector<std::string> strs;
  cudaError_t ce = cudaMemcpyAsync(d_ptrs, ptrs.data(), ptrs.size() * 8, cudaMemcpyHostToDevice, p->stream);
  int rc = ce == cudaSuccess ? fetch_string_records(p->stream, d_ptrs, (int64_t)ptrs.size(), 1, strs) : set_error(SD_ERR_CUDA, "cudaMemcpyAsync: %s", cudaGetErrorString(ce));
  cudaFree(d_ptrs);
  if (rc) return rc;
  for (size_t i = 0; i < ptrs.size(); i++) out[(uint64_t)ptrs[i]] = strs[i];
  return 0;
}

// compacted entries of a hash group table on the device: keys [count][nk], knull, vals [count][ns], K words [count][nsh]
struct Entries {
  int64_t* keys = nullptr; uint32_t* knull = nullptr; uint64_t* vals = nullptr; uint64_t* shifts = nullptr; uint32_t* cursor = nullptr;
  uint32_t count = 0;
  void release() {
    if (keys) cudaFree(keys);
    if (knull) cudaFree(knull);
    if (vals) cudaFree(vals);
    if (shifts) cudaFree(shifts);
    if (cursor) cudaFree(cursor);
    *this = Entries();
  }
};
int compact_entries(sd_plan* p, const HashTable& t, uint32_t capacity, int nk, int ns, int nsh, uint32_t count, Entries& out) {
  const size_t n = std::max<uint32_t>(count, 1);
  out.count = count;
  SD_CUDA(cudaMalloc(&out.keys, n * std::max(nk, 1) * 8));
  SD_CUDA(cudaMalloc(&out.knull, n * 4));
  SD_CUDA(cudaMalloc(&out.vals, n * ns * 8));
  SD_CUDA(cudaMalloc(&out.cursor, 64));
  if (nsh) SD_CUDA(cudaMalloc(&out.shifts, n * nsh * 8));
  return hash_table_compact(p->stream, t, capacity, nk, ns, out.keys, out.knull, out.vals, out.cursor, nsh, out.shifts);
}

// compacted entries -> partial rows in p->finished_rows.  A key word is the value's code, the address of its record (STRING /
// wide DECIMAL keys of the hash table), or -- dict_keys, the roll-up of a dense table -- the query-global dictionary id of a
// STRING key.  Entries of a grouping-sets roll-up carry gid as their last key word.
int emit_entries(sd_plan* p, const Entries& d, int nk, bool dict_keys) {
  const PlanSpec& sp = p->spec;
  const int ns = (int)sp.slots.size(), nsh = (int)sp.shifts.size(), nscan = (int)sp.keys.size();
  const uint32_t count = d.count;
  std::vector<int64_t> hk((size_t)count * nk);
  std::vector<uint32_t> hn(count);
  std::vector<uint64_t> hv((size_t)count * ns), hs((size_t)count * nsh);
  if (count) {
    if (nsh) SD_CUDA(cudaMemcpyAsync(hs.data(), d.shifts, hs.size() * 8, cudaMemcpyDeviceToHost, p->stream));
    SD_CUDA(cudaMemcpyAsync(hk.data(), d.keys, hk.size() * 8, cudaMemcpyDeviceToHost, p->stream));
    SD_CUDA(cudaMemcpyAsync(hn.data(), d.knull, hn.size() * 4, cudaMemcpyDeviceToHost, p->stream));
    SD_CUDA(cudaMemcpyAsync(hv.data(), d.vals, hv.size() * 8, cudaMemcpyDeviceToHost, p->stream));
  }
  SD_CUDA(cudaStreamSynchronize(p->stream));
  // STRING keys are held by reference (address of the [len][bytes] record in a resident buffer): fetch their bytes
  std::vector<std::vector<std::string>> key_strings((size_t)nk);
  for (int k = 0; k < nscan && count && !dict_keys; k++) {
    if (sp.exprs[sp.keys[k]].type != SD_STRING && !node_is_wide(sp, sp.keys[k])) continue;
    int rc = fetch_string_records(p->stream, d.keys + k, (int64_t)count, nk, key_strings[(size_t)k]);
    if (rc) return rc;
  }
  const std::vector<int> types = partial_field_types(sp);
  StrMap agg_strs;
  int rc = fetch_agg_strings(p, hv.data(), count, agg_strs);
  if (rc) return rc;
  std::vector<uint8_t>& out = p->finished_rows;
  out.clear();
  for (uint32_t g = 0; g < count; g++) {
    std::vector<HVal> vals;
    for (int k = 0; k < nk; k++) {
      HVal v;
      const int64_t code = hk[(size_t)g * nk + k];
      if ((hn[g] >> k) & 1u) v.isnull = true;
      else if (dict_keys && k < nscan) v.s = p->key_vals[(size_t)k][(size_t)code];
      else if (types[k] == SD_STRING) v.s = key_strings[(size_t)k][g];
      else if (!key_strings[(size_t)k].empty()) {   // wide DECIMAL key held by reference
        const std::string& b = key_strings[(size_t)k][g];
        if (b.empty() || b.size() > 16) return set_error(SD_ERR_CUDA, "corrupt DECIMAL key record (%zu bytes)", b.size());
        v.w = dec_from_bytes(reinterpret_cast<const uint8_t*>(b.data()), b.size()); v.i = (int64_t)v.w;
      }
      else if (type_is_fp(types[k])) memcpy(&v.d, &code, 8);
      else { v.i = code; v.w = code; }
      vals.push_back(v);
    }
    append_agg_fields(sp, &hv[(size_t)g * ns], nsh ? &hs[(size_t)g * nsh] : nullptr, vals, &agg_strs);
    emit_unsafe_row(out, types, vals);
  }
  p->finished_nrows = count;
  return 0;
}

// grouping sets: the fine groups in `a` (compacted hash entries, or the dense table when a.keys is null) rolled up into
// (keys, gid) on the device, then emitted.  The roll-up table starts at 2 x fine x sets entries -- a bound on the coarse
// groups, so it overflows only when an insert exhausts its probe budget; it then grows and the roll-up runs again (the scan is
// not replayed).
int rollup_rows(sd_plan* p, RollupArgs a, uint32_t fine_groups) {
  const PlanSpec& sp = p->spec;
  const int ns = (int)sp.slots.size(), nsh = (int)sp.shifts.size(), nk = (int)sp.keys.size();
  // the plan's tables: masks, slot ops, slot roles, per shift its n slot and S_j slots, per pair its two shifts
  std::vector<int32_t> meta;
  auto put = [&](const std::vector<int32_t>& v) { const size_t o = meta.size(); meta.insert(meta.end(), v.begin(), v.end()); return o; };
  std::vector<int32_t> masks(sp.sets.begin(), sp.sets.end()), ops(ns), roles(ns, -1);
  std::vector<int32_t> cnt((size_t)std::max(nsh, 1), 0), pows((size_t)std::max(nsh, 1) * 4, 0);
  std::vector<int32_t> px(std::max<size_t>(sp.pairs.size(), 1), 0), py(px.size(), 0);
  for (int s = 0; s < ns; s++) ops[s] = sp.slots[s].op;
  for (int i = 0; i < nsh; i++)
    for (int j = 1; j <= sp.shifts[i].order; j++) {
      roles[sp.shifts[i].pow_slot[j - 1]] = (i << 3) | j;
      pows[(size_t)i * 4 + j - 1] = sp.shifts[i].pow_slot[j - 1];
    }
  for (size_t q = 0; q < sp.pairs.size(); q++) { roles[sp.pairs[q].xy_slot] = -2 - (int)q; px[q] = sp.pairs[q].shift_x; py[q] = sp.pairs[q].shift_y; }
  for (auto& m : sp.agg_map) {   // n of a shift's input: its aggregate's count slot
    if (m.shift >= 0) cnt[m.shift] = m.count_slot;
    if (m.shift_y >= 0) cnt[m.shift_y] = m.count_slot;
  }
  const size_t o_masks = put(masks), o_ops = put(ops), o_roles = put(roles), o_cnt = put(cnt), o_pows = put(pows), o_px = put(px), o_py = put(py);
  if (meta.size() > p->rollup_meta_cap) {
    if (p->d_rollup_meta) cudaFree(p->d_rollup_meta);
    p->d_rollup_meta = nullptr;
    p->rollup_meta_cap = 0;
    SD_CUDA(cudaMalloc(&p->d_rollup_meta, meta.size() * 4));
    p->rollup_meta_cap = meta.size();
  }
  SD_CUDA(cudaMemcpyAsync(p->d_rollup_meta, meta.data(), meta.size() * 4, cudaMemcpyHostToDevice, p->stream));
  a.masks = reinterpret_cast<const uint32_t*>(p->d_rollup_meta + o_masks);
  a.slot_op = p->d_rollup_meta + o_ops; a.slot_role = p->d_rollup_meta + o_roles;
  a.shift_count = p->d_rollup_meta + o_cnt; a.shift_pow = p->d_rollup_meta + o_pows;
  a.pair_x = p->d_rollup_meta + o_px; a.pair_y = p->d_rollup_meta + o_py;
  a.nk = nk; a.ns = ns; a.nsh = nsh; a.nsets = (int)sp.sets.size(); a.rows_slot = sp.rows_slot;
  int rc = hash_ident(p);
  if (rc) return rc;
  constexpr uint32_t CAP_MAX = 1u << 28;
  const uint64_t want = std::max<uint64_t>(2ull * a.nfine * (uint64_t)a.nsets, 1024);
  uint32_t cap = 1024;
  while (cap < want && cap < CAP_MAX) cap *= 2;
  if (const char* e = getenv("SD_TUNE_ROLLUP_CAP")) {   // first capacity (tests: the growth path)
    const long v = atol(e);
    if (v >= 16 && (v & (v - 1)) == 0 && v <= (long)CAP_MAX) cap = (uint32_t)v;
  }
  double ms = 0;
  int launches = 0;
  uint32_t flags[16];
  for (;;) {
    if (cap != p->rollup_capacity) {
      p->rollup_capacity = 0;
      rc = table_alloc(p->rollup, cap, nk + 1, ns, nsh);
      if (rc) return rc;
      p->rollup_capacity = cap;
    }
    rc = hash_table_init(p->stream, p->rollup, cap, ns, p->d_hash_ident, nsh);
    if (rc) return rc;
    a.out = p->rollup;
    if (!p->ev_rollup[0]) { SD_CUDA(cudaEventCreate(&p->ev_rollup[0])); SD_CUDA(cudaEventCreate(&p->ev_rollup[1])); }
    SD_CUDA(cudaEventRecord(p->ev_rollup[0], p->stream));
    rc = rollup_launch(p->stream, a);
    if (rc) return rc;
    SD_CUDA(cudaEventRecord(p->ev_rollup[1], p->stream));
    launches++;
    SD_CUDA(cudaMemcpyAsync(flags, p->rollup.overflow, 64, cudaMemcpyDeviceToHost, p->stream));
    SD_CUDA(cudaStreamSynchronize(p->stream));
    float lms = 0;
    if (cudaEventElapsedTime(&lms, p->ev_rollup[0], p->ev_rollup[1]) == cudaSuccess) ms += lms;
    if (!flags[0]) break;
    if (cap >= CAP_MAX) return set_error(SD_ERR_UNSUPPORTED, "grouping-sets roll-up table would exceed 2^28 entries");
    cap *= 2;
  }
  Entries c;
  rc = compact_entries(p, p->rollup, p->rollup_capacity, nk + 1, ns, nsh, flags[8], c);
  if (rc) { c.release(); return rc; }
  p->rollup_info[0] = ms; p->rollup_info[1] = fine_groups; p->rollup_info[2] = flags[8]; p->rollup_info[3] = launches;
  rc = emit_entries(p, c, nk + 1, a.keys == nullptr);
  c.release();
  return rc;
}

// MODE_HASH: grow + replay on overflow, compact the occupied entries, emit partial rows
int finish_hash(sd_plan* p) {
  const PlanSpec& sp = p->spec;
  const int ns = (int)sp.slots.size(), nk = (int)sp.keys.size(), nsh = (int)sp.shifts.size();
  if (!p->hash_capacity) { int rc = hash_ensure(p, 1u << 16); if (rc) return rc; }
  uint32_t flags[16];
  for (;;) {
    SD_CUDA(cudaMemcpyAsync(flags, p->hash.overflow, 64, cudaMemcpyDeviceToHost, p->stream));
    SD_CUDA(cudaStreamSynchronize(p->stream));
    const uint32_t overflow = flags[0], count = flags[8];
    if (!overflow && (uint64_t)count * 2 <= p->hash_capacity) break;
    // too full (or an insert gave up): grow and replay every launch of this execution over the same bytes
    if (p->hash_capacity >= (1u << 28)) return set_error(SD_ERR_UNSUPPORTED, "group-by hash table would exceed 2^28 entries");
    uint32_t ncap = p->hash_capacity * 8;
    while ((uint64_t)count * 4 > ncap && ncap < (1u << 28)) ncap *= 2;
    int rc = hash_ensure(p, ncap);
    if (rc) return rc;
    SD_CUDA(cudaMemsetAsync(p->d_counters, 0, 64, p->stream));
    p->replay_kind = SDX_REPLAY_HASH_GROW;
    for (auto& l : p->launch_log) { rc = launch_scan(p, l.d_batches, l.d_prefix, l.nbatches, l.total_chunks, l.needs_slow, l.paths, nullptr, l.batch_base); if (rc) return rc; }
    p->replay_kind = SDX_REPLAY_NONE;
  }
  const uint32_t count = flags[8];
  Entries f;
  int rc = compact_entries(p, p->hash, p->hash_capacity, nk, ns, nsh, count, f);
  if (rc) return rc;
  unsigned long long counters[2] = {0, 0};
  SD_CUDA(cudaMemcpyAsync(counters, p->d_counters, 16, cudaMemcpyDeviceToHost, p->stream));
  SD_CUDA(cudaStreamSynchronize(p->stream));
  if (getenv("SD_DEBUG_VERIFY")) {   // diagnostic builds (SD_JIT_DEFINES=-DSD_EXP_VERIFY=1): staged tile vs global memory
    unsigned long long dbg[8] = {0};
    SD_CUDA(cudaMemcpy(dbg, p->d_counters, 64, cudaMemcpyDeviceToHost));
    uint32_t hist[64] = {0};
    SD_CUDA(cudaMemcpy(hist, p->hash.overflow, 256, cudaMemcpyDeviceToHost));
    SD_CUDA(cudaMemset(p->hash.overflow + 16, 0, 192));
    fprintf(stderr, "[verify] by consumer warp:");
    for (int i = 0; i < 8; i++) fprintf(stderr, " %u", hist[16 + i]);
    fprintf(stderr, "   by eighth of the tile (128 rows each):");
    for (int i = 0; i < 8; i++) fprintf(stderr, " %u", hist[24 + i]);
    fprintf(stderr, "   by column:");
    for (int i = 0; i < 4; i++) fprintf(stderr, " %u", hist[32 + i]);
    fprintf(stderr, "   tiles with any mismatch (warp-level): %u of %u warp-tiles\n", hist[40], hist[41]);
    fprintf(stderr, "[verify] of the mismatches: %llu = the stage's PREVIOUS occupant (read before the copy landed), %llu = its NEXT occupant (overwritten before the read)\n", dbg[2], dbg[3]);
    fprintf(stderr, "[verify] mismatching values %llu; first: column %llu stage %llu row %llu staged %016llx true %016llx\n", dbg[4],
            (dbg[5] >> 56) - (dbg[5] ? 1 : 0), (dbg[5] >> 48) & 0xff, dbg[5] & 0xffffffffffffull, dbg[6], dbg[7]);
  }
  update_agg_time(p);
  p->metrics[6] = (int64_t)(p->agg_ms * 1e6);
  p->metrics[8] = (int64_t)counters[0];
  p->metrics[11] = (int64_t)counters[0];
  if (!sp.sets.empty()) {
    RollupArgs a;
    memset(&a, 0, sizeof(a));
    a.keys = f.keys; a.knull = f.knull; a.vals = f.vals; a.shifts = f.shifts;
    a.nfine = count;
    for (int k = 0; k < nk; k++)
      if (sp.exprs[sp.keys[k]].type == SD_STRING || node_is_wide(sp, sp.keys[k])) a.strmask |= 1u << k;
    rc = rollup_rows(p, a, count);
    f.release();
    return rc;
  }
  rc = emit_entries(p, f, nk, false);
  f.release();
  return rc;
}

// MODE_PROJECT: grow + replay when the record buffer was too small, then records -> UnsafeRows
// The projected rows built by the GPU (sd_rows.cu).  *done = false: this execution needs the host writer below (more than 32
// fields, or a projected STRING column whose dictionary has entries that exist only on the host: values brought by an update
// delta).
static int project_rows_on_device(sd_plan* p, unsigned long long count, bool* done) {
  *done = false;
  const bool off = getenv("SD_TUNE_HOST_ROWS") != nullptr;   // (tests compare the two writers byte for byte)
  const PlanSpec& sp = p->spec;
  const int np = (int)sp.proj.size();
  if (off || np > ROW_MAX_FIELDS || count >= (1ull << 31) - 2) return 0;
  uint8_t kinds[ROW_MAX_FIELDS];
  std::vector<int> str_cols;
  for (int j = 0; j < np; j++) {
    const sd_expr& e = sp.exprs[sp.proj[j]];
    if (node_is_wide(sp, sp.proj[j])) return 0;   // wide DECIMAL records: the host writer below
    switch (e.type) {
      case SD_BOOLEAN: kinds[j] = ROW_KIND_BOOL; break;
      case SD_BYTE: kinds[j] = ROW_KIND_1; break;
      case SD_SHORT: kinds[j] = ROW_KIND_2; break;
      case SD_INT: case SD_DATE: kinds[j] = ROW_KIND_4; break;
      case SD_FLOAT: kinds[j] = ROW_KIND_FLOAT; break;
      case SD_STRING: kinds[j] = ROW_KIND_STRING; str_cols.push_back(e.a); break;
      default: kinds[j] = ROW_KIND_8; break;
    }
  }
  RowWriterBuffers& b = p->roww;
  const int ns = (int)str_cols.size(), nb = (int)p->exec_batches.size();
  if (ns > 0) {
    std::vector<const void*> key;
    key.reserve((size_t)nb + 1);
    key.push_back(reinterpret_cast<const void*>((uintptr_t)ns));
    for (const StoredBatch* sb : p->exec_batches) key.push_back(reinterpret_cast<const void*>((uintptr_t)sb->uid));
    if (key != b.src_key || !b.d_src) {
      b.src_key.clear();
      std::vector<RowStrSrc> src((size_t)nb * ns);
      std::vector<int32_t> recoff;
      std::vector<size_t> first((size_t)nb * ns, SIZE_MAX);
      for (int bi = 0; bi < nb; bi++) {
        const StoredBatch& sb = *p->exec_batches[bi];
        for (int k = 0; k < ns; k++) {
          const StoredCol& sc = sb.cols[sb.positional ? str_cols[k] : sp.cols[str_cols[k]].table_ordinal];
          RowStrSrc& r = src[(size_t)bi * ns + k];
          if (sc.raw_str) { r = RowStrSrc{sc.dev.dict, nullptr, -1, 0}; continue; }
          if (sc.dict_rec_off.size() != sc.dict_strings.size() || !sc.dev_base) return 0;   // host-only dictionary entries
          first[(size_t)bi * ns + k] = recoff.size();
          for (int64_t o : sc.dict_rec_off) {
            if (o < 0 || o > INT32_MAX) return 0;
            recoff.push_back((int32_t)o);
          }
          r = RowStrSrc{sc.dev_base, nullptr, sc.dev.dict_n, (int32_t)sc.dict_strings.size()};
        }
      }
      if (recoff.size() * 4 > b.recoff_cap) {
        if (b.d_recoff) cudaFree(b.d_recoff);
        b.d_recoff = nullptr; b.recoff_cap = 0;
        SD_CUDA(cudaMalloc(reinterpret_cast<void**>(&b.d_recoff), recoff.size() * 4 + 4096));
        b.recoff_cap = recoff.size() * 4 + 4096;
      }
      if (src.size() * sizeof(RowStrSrc) > b.src_cap) {
        if (b.d_src) cudaFree(b.d_src);
        b.d_src = nullptr; b.src_cap = 0;
        SD_CUDA(cudaMalloc(reinterpret_cast<void**>(&b.d_src), src.size() * sizeof(RowStrSrc) + 4096));
        b.src_cap = src.size() * sizeof(RowStrSrc) + 4096;
      }
      for (size_t i = 0; i < src.size(); i++) if (first[i] != SIZE_MAX) src[i].rec_off = b.d_recoff + first[i];
      // (pageable sources: both copies are staged by the driver before the calls return)
      if (!recoff.empty()) SD_CUDA(cudaMemcpyAsync(b.d_recoff, recoff.data(), recoff.size() * 4, cudaMemcpyHostToDevice, p->stream));
      SD_CUDA(cudaMemcpyAsync(b.d_src, src.data(), src.size() * sizeof(RowStrSrc), cudaMemcpyHostToDevice, p->stream));
      SD_CUDA(cudaStreamSynchronize(p->stream));
      b.src_key.swap(key);
    }
  }
  int64_t total = 0;
  int rc = device_write_rows(p->stream, reinterpret_cast<const uint64_t*>(p->d_out), (int64_t)count, np, kinds, nb, b, &total);
  if (rc) return rc;
  unsigned long long counters[2] = {0, 0};
  SD_CUDA(cudaMemcpyAsync(counters, p->d_counters, 16, cudaMemcpyDeviceToHost, p->stream));
  SD_CUDA(cudaStreamSynchronize(p->stream));
  update_agg_time(p);
  p->metrics[6] = (int64_t)(p->agg_ms * 1e6);
  p->metrics[8] = (int64_t)counters[0];
  p->metrics[11] = (int64_t)counters[0];
  p->finished_rows.clear();
  p->dev_rows_len = total;
  p->finished_nrows = (int64_t)count;
  *done = true;
  return 0;
}

// rows of this execution on the host (callers that post-process them: the exchange, the partial merge)
static int rows_to_host(sd_plan* p) {
  if (p->dev_rows_len < 0) return 0;
  p->finished_rows.resize((size_t)p->dev_rows_len);
  if (p->dev_rows_len) SD_CUDA(cudaMemcpyAsync(p->finished_rows.data(), p->roww.d_rows, (size_t)p->dev_rows_len, cudaMemcpyDeviceToHost, p->stream));
  SD_CUDA(cudaStreamSynchronize(p->stream));
  p->dev_rows_len = -1;
  return 0;
}

int finish_project(sd_plan* p) {
  const PlanSpec& sp = p->spec;
  const int np = (int)sp.proj.size();
  const int64_t rec = 8 + 8 * (int64_t)np;
  int rc = ensure_out(p, p->out_cap ? p->out_cap : 1024);
  if (rc) return rc;
  unsigned long long count = 0;
  for (;;) {
    SD_CUDA(cudaMemcpyAsync(&count, p->d_out_count, 8, cudaMemcpyDeviceToHost, p->stream));
    SD_CUDA(cudaStreamSynchronize(p->stream));
    if ((int64_t)count <= p->out_cap) break;
    rc = ensure_out(p, (int64_t)count + (int64_t)count / 8 + 1024);
    if (rc) return rc;
    SD_CUDA(cudaMemsetAsync(p->d_out_count, 0, 8, p->stream));
    SD_CUDA(cudaMemsetAsync(p->d_counters, 0, 64, p->stream));
    p->replay_kind = SDX_REPLAY_ROWS_GROW;
    for (auto& l : p->launch_log) { rc = launch_scan(p, l.d_batches, l.d_prefix, l.nbatches, l.total_chunks, l.needs_slow, l.paths, nullptr, l.batch_base); if (rc) return rc; }
    p->replay_kind = SDX_REPLAY_NONE;
  }
  {
    bool done = false;
    rc = project_rows_on_device(p, count, &done);
    if (rc || done) return rc;
  }
  static const bool dbg = getenv("SD_DEBUG_TIMING") != nullptr;
  const auto t_begin = std::chrono::steady_clock::now();
  auto lap = [&](const char* what) { if (dbg) fprintf(stderr, "[finish_project] %s at %.2f ms\n", what, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_begin).count()); };
  // (page-locked staging for the records: a pageable destination makes the driver bounce the copy through its own buffers)
  const size_t rec_bytes = (size_t)count * (size_t)rec;
  if (rec_bytes > p->h_recs_cap) {
    if (p->h_recs) cudaFreeHost(p->h_recs);
    p->h_recs = nullptr; p->h_recs_cap = 0;
    SD_CUDA(cudaMallocHost(&p->h_recs, rec_bytes + rec_bytes / 4 + 4096));
    p->h_recs_cap = rec_bytes + rec_bytes / 4 + 4096;
  }
  const uint64_t* recs = p->h_recs;
  unsigned long long counters[2] = {0, 0};
  if (count) SD_CUDA(cudaMemcpyAsync(p->h_recs, p->d_out, rec_bytes, cudaMemcpyDeviceToHost, p->stream));
  SD_CUDA(cudaMemcpyAsync(counters, p->d_counters, 16, cudaMemcpyDeviceToHost, p->stream));
  SD_CUDA(cudaStreamSynchronize(p->stream));
  update_agg_time(p);
  p->metrics[6] = (int64_t)(p->agg_ms * 1e6);
  p->metrics[8] = (int64_t)counters[0];
  p->metrics[11] = (int64_t)counters[0];
  std::vector<int> types;
  std::vector<int> str_col(np, -1);
  std::vector<char> wide(np, 0);   // wide DECIMAL column: the record holds the device address of its [len][bytes] record
  for (int j = 0; j < np; j++) {
    const sd_expr& e = sp.exprs[sp.proj[j]];
    types.push_back(field_type(e.type, e.type == SD_DECIMAL ? decimal_ps(sp, sp.proj[j]) : 0));
    if (e.type == SD_STRING) str_col[j] = e.a;
    wide[j] = node_is_wide(sp, sp.proj[j]);
  }
  lap("records on the host");
  // strings of raw (variable-width) batches are projected by reference: record = position in the batch's body
  std::vector<int64_t> raw_ptrs;
  for (unsigned long long i = 0; i < count && !str_col.empty(); i++) {
    const uint64_t* r = &recs[(size_t)i * (size_t)(rec / 8)];
    const uint32_t bidx = (uint32_t)(r[0] & 0xffffffffu), pnull = (uint32_t)(r[0] >> 32);
    if (bidx >= p->exec_batches.size()) return set_error(SD_ERR_CUDA, "corrupt projection record (batch %u)", bidx);
    const StoredBatch& sb = *p->exec_batches[bidx];
    for (int j = 0; j < np; j++) {
      if (wide[j] && !((pnull >> j) & 1u)) { raw_ptrs.push_back((int64_t)r[1 + j]); continue; }
      if (str_col[j] < 0 || ((pnull >> j) & 1u)) continue;
      const StoredCol& sc = sb.cols[sb.positional ? str_col[j] : sp.cols[str_col[j]].table_ordinal];
      if (sc.raw_str) raw_ptrs.push_back((int64_t)(uintptr_t)(sc.dev.dict + (uint32_t)r[1 + j]));
    }
  }
  std::vector<std::string> raw_strings;
  if (!raw_ptrs.empty()) {
    int64_t* d_ptrs = nullptr;
    SD_CUDA(cudaMalloc(&d_ptrs, raw_ptrs.size() * 8));
    cudaError_t ce = cudaMemcpyAsync(d_ptrs, raw_ptrs.data(), raw_ptrs.size() * 8, cudaMemcpyHostToDevice, p->stream);
    rc = ce == cudaSuccess ? fetch_string_records(p->stream, d_ptrs, (int64_t)raw_ptrs.size(), 1, raw_strings) : set_error(SD_ERR_CUDA, "cudaMemcpyAsync: %s", cudaGetErrorString(ce));
    cudaFree(d_ptrs);
    if (rc) return rc;
  }
  // records -> UnsafeRows, written in place (no per-row value objects: C4 emits ~1 M rows per execution)
  size_t next_raw = 0;
  std::vector<uint8_t>& out = p->finished_rows;
  out.clear();
  const int64_t bits = ((np + 63) / 64) * 8, fixed = bits + 8 * (int64_t)np;
  // pass 1: sizes (strings are the only variable part)
  size_t total = 0;
  {
    size_t nr = 0;
    for (unsigned long long i = 0; i < count; i++) {
      const uint64_t* r = &recs[(size_t)i * (size_t)(rec / 8)];
      const uint32_t bidx = (uint32_t)(r[0] & 0xffffffffu), pnull = (uint32_t)(r[0] >> 32);
      const StoredBatch& sb = *p->exec_batches[bidx];
      int64_t var = 0;
      for (int j = 0; j < np; j++) {
        if (wide[j]) { var += 16; if (!((pnull >> j) & 1u)) nr++; continue; }   // 16 bytes reserved even for NULL (emit_unsafe_row)
        if (str_col[j] < 0 || ((pnull >> j) & 1u)) continue;
        const StoredCol& sc = sb.cols[sb.positional ? str_col[j] : sp.cols[str_col[j]].table_ordinal];
        if (sc.raw_str) { var += ((int64_t)raw_strings[nr++].size() + 7) & ~int64_t(7); continue; }
        const int64_t code = (int64_t)r[1 + j];
        if (code == sc.dev.dict_n && code >= 0) continue;   // NULL code
        if (code < 0 || code >= (int64_t)sc.dict_strings.size()) return set_error(SD_ERR_CUDA, "dictionary code %lld out of range", (long long)code);
        var += ((int64_t)sc.dict_strings[(size_t)code].size() + 7) & ~int64_t(7);
      }
      total += (size_t)(8 + fixed + var);
    }
  }
  lap("sizes");
  out.assign(total, 0);
  lap("zero fill");
  uint8_t* w = out.data();
  for (unsigned long long i = 0; i < count; i++) {
    const uint64_t* r = &recs[(size_t)i * (size_t)(rec / 8)];
    const uint32_t bidx = (uint32_t)(r[0] & 0xffffffffu), pnull = (uint32_t)(r[0] >> 32);
    const StoredBatch& sb = *p->exec_batches[bidx];
    uint8_t* row = w + 8;
    int64_t voff = fixed;
    for (int j = 0; j < np; j++) {
      uint8_t* slot = row + bits + 8 * (int64_t)j;
      if (wide[j]) {   // (offset << 32 | size) + the record's BigInteger bytes in a 16-byte region
        int64_t ol = voff << 32;
        if ((pnull >> j) & 1u) row[j >> 3] |= (uint8_t)(1u << (j & 7));
        else {
          const std::string& b = raw_strings[next_raw++];
          if (b.empty() || b.size() > 16) return set_error(SD_ERR_CUDA, "corrupt DECIMAL record (%zu bytes)", b.size());
          memcpy(row + voff, b.data(), b.size());
          ol |= (int64_t)b.size();
        }
        memcpy(slot, &ol, 8);
        voff += 16;
        continue;
      }
      if ((pnull >> j) & 1u) { row[j >> 3] |= (uint8_t)(1u << (j & 7)); continue; }
      const uint64_t raw = r[1 + j];
      const int t = ft_base(types[j]);
      if (t == SD_STRING) {
        const StoredCol& sc = sb.cols[sb.positional ? str_col[j] : sp.cols[str_col[j]].table_ordinal];
        const std::string* sv;
        if (sc.raw_str) sv = &raw_strings[next_raw++];
        else {
          const int64_t code = (int64_t)raw;
          if (code == sc.dev.dict_n) { row[j >> 3] |= (uint8_t)(1u << (j & 7)); continue; }
          sv = &sc.dict_strings[(size_t)code];
        }
        const int64_t ol = (voff << 32) | (int64_t)sv->size();
        memcpy(slot, &ol, 8);
        memcpy(row + voff, sv->data(), sv->size());
        voff += ((int64_t)sv->size() + 7) & ~int64_t(7);
        continue;
      }
      switch (t) {
        case SD_BOOLEAN: slot[0] = raw != 0; break;
        case SD_BYTE: memcpy(slot, &raw, 1); break;
        case SD_SHORT: memcpy(slot, &raw, 2); break;
        case SD_INT: case SD_DATE: memcpy(slot, &raw, 4); break;
        case SD_FLOAT: { double d; memcpy(&d, &raw, 8); const float f = (float)d; memcpy(slot, &f, 4); break; }
        default: memcpy(slot, &raw, 8); break;   // LONG, TIMESTAMP, DOUBLE (its bits), DECIMAL(p <= 18)
      }
    }
    const int64_t sz = voff;
    memcpy(w, &sz, 8);
    w += 8 + sz;
  }
  lap("rows written");
  p->finished_nrows = (int64_t)count;
  return 0;
}

int ensure_private_store(sd_plan* p) {
  if (p->priv) return 0;
  // the private store's "table" is exactly the plan's scan columns
  std::vector<sd_column> schema(p->spec.cols);
  return sd_store_create(p->device, (int32_t)schema.size(), schema.data(), &p->priv);
}

}  // namespace

extern "C" {

int sd_init(int device) {
  int n = 0;
  SD_CUDA(cudaGetDeviceCount(&n));
  if (device < 0 || device >= n) return set_error(SD_ERR_INVALID, "sd_init: device %d of %d", device, n);
  SD_CUDA(cudaSetDevice(device));
  t_device = device;
  return 0;
}
int sd_device_count(int* out) { SD_CUDA(cudaGetDeviceCount(out)); return 0; }
const char* sd_version(void) { return "snappydata_b200 0.1.0 (sm_90a)"; }

int sdx_stats_pass(const sd_plan_desc* desc, const sd_literal* lits, int32_t nlits, const void* stats, int64_t stats_len,
                   int32_t stats_ncols, int32_t num_rows, int32_t* pass) {
  return stats_pass_hook(desc, lits, nlits, stats, stats_len, stats_ncols, num_rows, pass);
}

int sd_plan_create(const sd_plan_desc* desc, sd_plan** out) {
  if (!out) return set_error(SD_ERR_INVALID, "sd_plan_create: null out");
  std::unique_ptr<sd_plan, void (*)(sd_plan*)> p(new sd_plan(), sd_plan_destroy);   // a failure below releases what was created
  std::string err;
  int rc = analyze_plan(desc, p->spec, err);
  if (rc) return set_error(rc, "sd_plan_create: %s", err.c_str());
  p->device = t_device;
  SD_CUDA(cudaSetDevice(p->device));
  // kernel: ahead-of-time compiled plan, else NVRTC
  {
    CodegenOptions opt;
    sd_plan_desc dv = p->spec.desc_view();
    rc = resolve_kernel(dv, opt, p->device, &p->kernel, nullptr);
    if (rc) return rc;
    p->active = &p->kernel;
  }
  p->kernel_name = p->kernel.origin + ":" + p->kernel.name;
  cudaDeviceProp prop;
  SD_CUDA(cudaGetDeviceProperties(&prop, p->device));
  p->num_sms = prop.multiProcessorCount;
  p->smem_optin = (int)prop.sharedMemPerBlockOptin;
  SD_CUDA(cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking));
  p->own_stream = true;
  SD_CUDA(cudaEventCreate(&p->ev_start));
  SD_CUDA(cudaEventCreate(&p->ev_stop));
  SD_CUDA(cudaMalloc(&p->d_ticket, 64));
  SD_CUDA(cudaMemset(p->d_ticket, 0, 64));
  rc = ensure_result(p.get(), 64);   // d_state: counters + room for a small group table
  if (rc) return rc;
  p->scratch.device = p->device;
  p->scratch.slab_bytes = size_t(8) << 20;
  p->cache_arena.device = p->device;
  p->cache_arena.slab_bytes = size_t(8) << 20;
  const int nk = (int)p->spec.keys.size();
  p->key_ids.resize(nk);
  p->key_vals.resize(nk);
  p->key_null_id.assign(nk, -1);
  p->lits.resize(p->spec.literal_types.size());
  p->lit_strs.resize(p->spec.literal_types.size());
  for (size_t i = 0; i < p->lits.size(); i++) { memset(&p->lits[i], 0, sizeof(sd_literal)); p->lits[i].type = p->spec.literal_types[i]; }
  if (p->spec.mode == MODE_GROUPS) p->chunk_rows = 2 * CHUNK_ROWS;   // tools/sweep.sh measures it
  if (const char* e = getenv("SD_TUNE_CHUNK_ROWS")) { int v = atoi(e); if (v >= 2048 && v % 2048 == 0 && v <= (1 << 20)) p->chunk_rows = v; }
  p->lits_set = p->lits.empty();
  *out = p.release();
  return 0;
}

int sd_plan_set_literals(sd_plan* p, const sd_literal* vals, int32_t n) {
  if (!p) return set_error(SD_ERR_INVALID, "null plan");
  if (n != (int)p->lits.size()) return set_error(SD_ERR_INVALID, "sd_plan_set_literals: plan has %zu literal slots, got %d", p->lits.size(), n);
  if (!p->pending.empty()) return set_error(SD_ERR_STATE, "sd_plan_set_literals: batches already submitted for this execution");
  for (int i = 0; i < n; i++)
    if (p->spec.lit_wide[(size_t)i] && !vals[i].is_null && (!vals[i].s || vals[i].slen < 1 || vals[i].slen > 16))
      return set_error(SD_ERR_INVALID, "sd_plan_set_literals: slot %d holds a DECIMAL wider than 18 digits: its value needs 1..16 bytes (BigInteger.toByteArray)", i);
  for (int i = 0; i < n; i++) {
    p->lits[i] = vals[i];
    p->lit_strs[i].assign(vals[i].s ? vals[i].s : "", vals[i].s ? (size_t)std::max(0, vals[i].slen) : 0);
    p->lits[i].s = p->lit_strs[i].data();
    p->lits[i].slen = (int32_t)p->lit_strs[i].size();
  }
  p->lits_set = true;
  p->litpool_dirty = true;
  return 0;
}

int sd_plan_set_option(sd_plan* p, int32_t option, int64_t value) {
  if (!p) return set_error(SD_ERR_INVALID, "null plan");
  if (option == SD_OPT_RETAIN_BUFFERS) {
    int rc = ensure_private_store(p);
    if (rc) return rc;
    p->priv->retain_buffers = value != 0;
    return 0;
  }
  return set_error(SD_ERR_INVALID, "unknown option %d", option);
}

int sd_plan_set_stream(sd_plan* p, void* cuda_stream) {
  if (!p) return set_error(SD_ERR_INVALID, "null plan");
  if (p->own_stream && p->stream) { cudaSetDevice(p->device); cudaStreamDestroy(p->stream); }
  p->stream = reinterpret_cast<cudaStream_t>(cuda_stream);
  p->own_stream = false;
  return 0;
}

const char* sd_plan_kernel_name(sd_plan* p) { return p ? p->kernel_name.c_str() : ""; }

int sd_batch_submit(sd_plan* p, const sd_batch* b) {
  if (!p || !b) return set_error(SD_ERR_INVALID, "sd_batch_submit: null argument");
  if (!p->lits_set) return set_error(SD_ERR_STATE, "sd_batch_submit: literals not set");
  if (p->spec.mode == MODE_MUTATE) return set_error(SD_ERR_STATE, "sd_batch_submit: an UPDATE / DELETE plan runs over a resident store only");
  if (b->ncols != (int)p->spec.cols.size()) return set_error(SD_ERR_INVALID, "sd_batch_submit: batch has %d columns, plan scans %zu", b->ncols, p->spec.cols.size());
  SD_CUDA(cudaSetDevice(p->device));
  p->metrics[2]++;   // columnBatchesSeen
  // stats-row skipping before any byte moves (ColumnTableScan.scala:532-543)
  if (b->stats_row && b->stats_len > 0 && p->spec.filter >= 0) {
    StatEval ev{p->spec, p->lits, reinterpret_cast<const uint8_t*>(b->stats_row), b->stats_len, 1 + 3 * b->stats_ncols, b->num_rows};
    Tri r;
    if (ev.eval(p->spec.filter, &r) && !r.isnull && !r.v) { p->metrics[5]++; return 0; }
  }
  int rc = ensure_private_store(p);
  if (rc) return rc;
  const int64_t before = p->priv->h2d_bytes;
  // the private store is indexed by scan column: buffers arrive in plan order already
  sd_batch local = *b;
  rc = store_put(p->priv, &local, nullptr);
  if (rc) return rc;
  p->metrics[10] += p->priv->h2d_bytes - before;
  p->priv->batches.back()->positional = true;
  const StoredBatch* sb = p->priv->batches.back().get();
  // scan columns of the private store are positional: re-point table ordinals on the fly in build_scan
  p->pending.push_back({sb});
  p->pending_bytes += p->priv->h2d_bytes - before;
  // (compressed inputs: one expansion launch per flush, as long as its longest buffer; the launches of successive
  // flushes overlap on their own streams, so the same flush size serves both)
  int64_t threshold = int64_t(256) << 20;
  if (const char* e = getenv("SD_TUNE_FLUSH_MB")) { const long v = atol(e); if (v >= 1 && v <= 65536) threshold = int64_t(v) << 20; }
  if (p->pending_bytes >= threshold) return flush_pending(p);
  return 0;
}

static int scan_store(sd_plan* p, sd_store* s, const int32_t* bucket_ids, int32_t nbuckets);

int sd_plan_scan_store(sd_plan* p, sd_store* s, const int32_t* bucket_ids, int32_t nbuckets) {
  if (!p || !s) return set_error(SD_ERR_INVALID, "sd_plan_scan_store: null argument");
  if (p->spec.mode == MODE_MUTATE) return set_error(SD_ERR_STATE, "sd_plan_scan_store: an UPDATE / DELETE plan runs through sd_plan_update_store / sd_plan_delete_store");
  return scan_store(p, s, bucket_ids, nbuckets);
}

}  // extern "C"

const PlanSpec& sd::plan_spec(const sd_plan* p) { return p->spec; }

// The scan of an UPDATE / DELETE statement (sd_mutate.cu merges what it finds): the plan's records over the store's current
// batches -- the same staged ring, overlay path, stats skipping and grow-and-replay as a projection -- left on the device.
int sd::mutation_scan(sd_plan* p, sd_store* s, const int32_t* bucket_ids, int32_t nbuckets, const sd_literal* lits, int32_t nlits,
                      MutationScan* out) {
  if (p->spec.mode != MODE_MUTATE) return set_error(SD_ERR_STATE, "not an UPDATE / DELETE plan (sd_plan_desc.flags lacks SD_PLAN_MUTATE)");
  int rc = sd_plan_reset(p);
  if (rc) return rc;
  rc = sd_plan_set_literals(p, lits, nlits);
  if (rc) return rc;
  rc = scan_store(p, s, bucket_ids, nbuckets);
  if (rc) return rc;
  rc = ensure_out(p, p->out_cap ? p->out_cap : 1024);
  if (rc) return rc;
  unsigned long long count = 0;
  for (;;) {   // the one read-back of the scan: how many rows matched (grow + replay when the record buffer was too small)
    SD_CUDA(cudaMemcpyAsync(&count, p->d_out_count, 8, cudaMemcpyDeviceToHost, p->stream));
    SD_CUDA(cudaStreamSynchronize(p->stream));
    if ((int64_t)count <= p->out_cap) break;
    rc = ensure_out(p, (int64_t)count + (int64_t)count / 8 + 1024);
    if (rc) return rc;
    SD_CUDA(cudaMemsetAsync(p->d_out_count, 0, 8, p->stream));
    SD_CUDA(cudaMemsetAsync(p->d_counters, 0, 64, p->stream));
    p->replay_kind = SDX_REPLAY_ROWS_GROW;
    for (auto& l : p->launch_log) { rc = launch_scan(p, l.d_batches, l.d_prefix, l.nbatches, l.total_chunks, l.needs_slow, l.paths, nullptr, l.batch_base); if (rc) return rc; }
    p->replay_kind = SDX_REPLAY_NONE;
  }
  update_agg_time(p);
  p->metrics[6] = (int64_t)(p->agg_ms * 1e6);
  out->records = reinterpret_cast<const uint64_t*>(p->d_out);
  out->count = (int64_t)count;
  out->rec_words = 2 + (int)std::max<size_t>(p->spec.proj.size(), 1);
  out->batches = p->exec_batches;
  out->stream = p->stream;
  out->scan_ms = p->agg_ms;
  p->finished_nrows = (int64_t)count;
  p->metrics[0] = (int64_t)count;
  // the statement goes on reading these batches, but under the store's mutate_mu, which keeps sd_store_reclaim out
  p->pins.release();
  return 0;
}

extern "C" {

static int scan_store(sd_plan* p, sd_store* s, const int32_t* bucket_ids, int32_t nbuckets) {
  if (!p->lits_set) return set_error(SD_ERR_STATE, "sd_plan_scan_store: literals not set");
  if (s->device != p->device) return set_error(SD_ERR_INVALID, "store lives on device %d, plan on %d", s->device, p->device);
  SD_CUDA(cudaSetDevice(p->device));
  int rc = flush_pending(p);
  if (rc) return rc;
  // snapshot under the store's lock: the batches present NOW are what this execution scans (ingest may continue meanwhile;
  // the reference's scan likewise sees the batches of its snapshot, ColumnFormatIterator over the bucket's entries)
  std::vector<const StoredBatch*> snapshot;
  int64_t snap_version;
  {
    std::lock_guard<std::mutex> lock(s->mu);
    rc = store_flush_lz4(s);
    if (rc) return rc;
    rc = store_lz4_check(s);   // resident stores: expansions happen once, before the first scan
    if (rc) return rc;
    snapshot.reserve(s->batches.size());
    for (auto& sbp : s->batches) snapshot.push_back(sbp.get());
    snap_version = s->version;
    p->pins.take(s->pins, snap_version);   // sd_store_reclaim frees nothing this snapshot can read until the pin is released
  }
  for (auto& c : p->spec.cols) {
    if (c.table_ordinal < 0 || c.table_ordinal >= (int)s->schema.size()) return set_error(SD_ERR_INVALID, "plan column ordinal %d outside the store schema", c.table_ordinal);
    const sd_column& sc = s->schema[c.table_ordinal];
    if (sc.type != c.type || sc.nullable != c.nullable)
      return set_error(SD_ERR_INVALID, "plan column %d (type %d nullable %d) does not match the store schema (type %d nullable %d)", c.table_ordinal,
                       c.type, c.nullable, sc.type, sc.nullable);
    // a DECIMAL of more than 18 digits is resident as record positions + body, a narrower one as int64 values: the kernel
    // reads the layout the PLAN's precision implies, so both sides must agree on it (and a wide column's scale on its values)
    if (c.type == SD_DECIMAL && (wide_decimal(c.type, c.precision) != wide_decimal(sc.type, sc.precision) ||
                                 (wide_decimal(c.type, c.precision) && c.scale != sc.scale)))
      return set_error(SD_ERR_INVALID, "plan column %d is DECIMAL(%d,%d), the store column DECIMAL(%d,%d): a DECIMAL of more than 18 digits "
                       "on one side only, or a different scale of one", c.table_ordinal, c.precision, c.scale, sc.precision, sc.scale);
  }
  std::vector<int32_t> buckets(bucket_ids, bucket_ids + (bucket_ids ? nbuckets : 0));
  const std::string lk = literal_key(p);
  sd_plan::ScanCache& c = p->cache;
  const bool same_query = c.valid && c.store == s && c.buckets == buckets && c.lit_key == lk;
  // descriptors (+ stats skipping, aux tables) of snapshot[from, end) as one segment in the cache arena
  auto build_segment = [&](size_t from, sd_plan::ScanSegment* seg, int64_t* seen, int64_t* skipped) -> int {
    std::vector<const StoredBatch*> list;
    for (size_t i = from; i < snapshot.size(); i++) {
      const StoredBatch& sb = *snapshot[i];
      if (!buckets.empty() && std::find(buckets.begin(), buckets.end(), sb.bucket_id) == buckets.end()) continue;
      if (sb.gone) continue;   // every row deleted (ColumnDelta.checkBatchDeleted): not a batch any more
      (*seen)++;
      if (!batch_passes_stats(p, sb)) { (*skipped)++; continue; }
      list.push_back(&sb);
    }
    BuiltScan bs;
    int rc2 = build_scan(p, list, p->cache_arena, p->stream, &bs);
    if (rc2) return rc2;
    // a key column without dictionary ids, or more key combinations than a dense table holds: the caller switches the plan
    // to the hash table and rebuilds every segment (descriptors built for the dense kernel carry key-id tables where the
    // hash kernel reads string-record addresses, so no segment built before the switch may be launched after it)
    if (p->spec.mode == MODE_GROUPS && (bs.needs_hash || dense_groups(p) > DENSE_GROUPS_MAX)) return -1000;
    seg->d_batches = bs.d_batches; seg->d_prefix = bs.d_prefix; seg->nbatches = bs.nbatches; seg->total_chunks = bs.total_chunks;
    seg->needs_slow = bs.needs_slow; seg->paths = bs.paths; seg->rows = bs.rows; seg->algo_bytes = bs.algo_bytes;
    seg->updated_cols = bs.updated_cols; seg->deleted_batches = bs.deleted_batches;
    seg->covered = snapshot.size() - from;
    seg->batches.swap(list);
    return 0;
  };
  bool rebuilt = false;
  if (same_query && c.version != snap_version && snapshot.size() >= c.snap_uids.size() && !getenv("SD_TUNE_NO_INCREMENTAL_SCAN")) {
    // the store changed: still the batches we know, plus new ones at the end?
    bool prefix = true;
    for (size_t i = 0; i < c.snap_uids.size() && prefix; i++) prefix = snapshot[i]->uid == c.snap_uids[i];
    if (prefix) {
      size_t from = c.snap_uids.size();
      // keep the tail short: fold the small segments after the first one into the new segment when there are several
      if (c.segs.size() > 4 && c.consolidations < 64) {
        size_t keep = c.segs[0].covered;
        c.segs.resize(1);
        // (seen / skipped of the folded segments are recounted by build_segment)
        int64_t seen0 = 0, skipped0 = 0;
        for (size_t i = 0; i < keep; i++) {
          const StoredBatch& sb = *snapshot[i];
          if (!buckets.empty() && std::find(buckets.begin(), buckets.end(), sb.bucket_id) == buckets.end()) continue;
          if (sb.gone) continue;
          seen0++;
        }
        skipped0 = seen0 - (int64_t)c.segs[0].batches.size();
        c.seen = seen0; c.skipped = skipped0;
        from = keep;
        c.consolidations++;
      }
      if (c.consolidations < 64) {
        sd_plan::ScanSegment seg;
        rc = build_segment(from, &seg, &c.seen, &c.skipped);
        if (rc == 0) {
          if (seg.covered) c.segs.push_back(std::move(seg));
          c.snap_uids.resize(snapshot.size());
          for (size_t i = from; i < snapshot.size(); i++) c.snap_uids[i] = snapshot[i]->uid;
          c.version = snap_version;
          rebuilt = true;
        } else if (rc != -1000) {
          return rc;
        }
      }
    }
  }
  // (the store's address and version do not identify its batches: a store created where a destroyed one lived starts at the
  // same version; batch uids are never reused)
  auto same_batches = [&]() {
    if (snapshot.size() != c.snap_uids.size()) return false;
    for (size_t i = 0; i < snapshot.size(); i++) if (snapshot[i]->uid != c.snap_uids[i]) return false;
    return true;
  };
  if (!rebuilt && !(same_query && c.version == snap_version && same_batches())) {
    // (re)build everything: stats skipping + descriptors + tables, kept on the device for repeated executions
    c.valid = false;
    c.segs.clear();
    c.consolidations = 0;
    p->cache_arena.reset();
    sd_plan::ScanSegment seg;
    int64_t seen = 0, skipped = 0;
    rc = build_segment(0, &seg, &seen, &skipped);
    if (rc == -1000) {
      rc = switch_to_hash(p);
      if (rc) return rc;
      p->cache_arena.reset();
      seen = skipped = 0;
      seg = sd_plan::ScanSegment();
      rc = build_segment(0, &seg, &seen, &skipped);
    }
    if (rc) return rc;
    c.store = s; c.version = snap_version; c.buckets = buckets; c.lit_key = lk;
    c.seen = seen; c.skipped = skipped;
    c.segs.push_back(std::move(seg));
    c.snap_uids.resize(snapshot.size());
    for (size_t i = 0; i < snapshot.size(); i++) c.snap_uids[i] = snapshot[i]->uid;
    c.valid = true;
  }
  p->metrics[2] += c.seen;
  p->metrics[5] += c.skipped;
  for (const sd_plan::ScanSegment& seg : c.segs) {
    p->metrics[3] += seg.updated_cols;
    p->metrics[4] += seg.deleted_batches;
    p->metrics[9] += seg.algo_bytes;
  }
  bool launched = false;
  for (const sd_plan::ScanSegment& seg : c.segs) {
    if (seg.nbatches == 0 && launched) continue;
    rc = launch_scan(p, seg.d_batches, seg.d_prefix, seg.nbatches, seg.total_chunks, seg.needs_slow, seg.paths, &seg.batches);
    if (rc) return rc;
    launched = true;
  }
  return 0;
}

// dense / no-key state (the [ngroups][slots] table the kernel leaves, then the K words [ngroups][shifts]) -> partial rows appended to `out`:
// UnsafeRow(group keys ++ aggregate buffers) (SnappyHashAggregateExec.scala:1148-1178).  The key dictionaries are arguments
// because the exchange's dense form carries ANOTHER rank's state and dictionaries (ids are private to a partition).
static int64_t dense_rows_from_state(const PlanSpec& sp, const uint64_t* h, int ngroups, const int32_t* radix, const std::vector<int>& key_null_id,
                                     const std::vector<std::vector<std::string>>& key_vals, const StrMap* agg_strs, std::vector<uint8_t>& out) {
  const int ns = (int)sp.slots.size(), nk = (int)sp.keys.size(), nsh = (int)sp.shifts.size();
  const std::vector<int> types = partial_field_types(sp);
  int64_t nrows = 0;
  std::vector<HVal> vals;
  for (int g = 0; g < ngroups; g++) {
    const uint64_t* sv = &h[(size_t)g * ns];
    if (nk > 0 && sv[sp.rows_slot] == 0) continue;   // group never seen
    vals.clear();
    int rem = g, idx[MAX_KEYS];
    for (int k = nk - 1; k >= 0; k--) { idx[k] = rem % radix[k]; rem /= radix[k]; }
    for (int k = 0; k < nk; k++) {
      HVal v;
      if (idx[k] == key_null_id[k]) v.isnull = true; else v.s = key_vals[k][idx[k]];
      vals.push_back(v);
    }
    append_agg_fields(sp, sv, nsh ? h + (size_t)ngroups * ns + (size_t)g * nsh : nullptr, vals, agg_strs);
    emit_unsafe_row(out, types, vals);
    nrows++;
  }
  return nrows;
}

// partial rows of this execution's dense / no-key result -> p->finished_rows
static int finish_dense(sd_plan* p) {
  const PlanSpec& sp = p->spec;
  const int ns = (int)sp.slots.size();
  int rc = 0;
  if (!p->result_init) { rc = init_result(p, 1); if (rc) return rc; p->ngroups = 1; }
  const size_t ne = (size_t)p->ngroups * ns;
  rc = ensure_result(p, result_words(sp, p->ngroups));
  if (rc) return rc;
  SD_CUDA(cudaMemcpyAsync(p->h_pinned, p->d_state, (STATE_HDR + result_words(sp, p->ngroups)) * 8, cudaMemcpyDeviceToHost, p->stream));   // counters + table in one copy
  SD_CUDA(cudaStreamSynchronize(p->stream));
  const uint64_t* h = p->h_pinned + STATE_HDR;
  const unsigned long long counters[2] = {p->h_pinned[0], p->h_pinned[1]};
  update_agg_time(p);
  p->metrics[6] = (int64_t)(p->agg_ms * 1e6);
  p->metrics[8] = (int64_t)counters[0];
  p->metrics[11] = (int64_t)counters[0];
  if (!sp.sets.empty()) {   // roll the dense table's groups up into (keys, gid)
    RollupArgs a;
    memset(&a, 0, sizeof(a));
    a.vals = p->d_result;
    a.shifts = p->d_result + (size_t)p->ngroups * ns;
    a.nfine = (uint32_t)p->ngroups;
    for (size_t k = 0; k < sp.keys.size(); k++) { a.radix[k] = p->radix[k]; a.null_id[k] = p->key_null_id[k]; }
    uint32_t fine = 0;
    for (int g = 0; g < p->ngroups; g++) fine += h[(size_t)g * ns + sp.rows_slot] != 0;
    return rollup_rows(p, a, fine);
  }
  StrMap agg_strs;
  {
    std::vector<uint64_t> copy(h, h + ne);   // (the pinned mirror is reused by the fetch's own read-backs)
    rc = fetch_agg_strings(p, copy.data(), (size_t)p->ngroups, agg_strs);
    if (rc) return rc;
  }
  std::vector<uint8_t>& out = p->finished_rows;
  out.clear();
  p->finished_nrows = dense_rows_from_state(sp, h, p->ngroups, p->radix, p->key_null_id, p->key_vals, &agg_strs, out);
  return 0;
}

// run what is pending and materialise this partition's partial rows in p->finished_rows (once per execution)
static int launch_what_is_pending(sd_plan* p) {
  SD_CUDA(cudaSetDevice(p->device));
  int rc = flush_pending(p);
  if (rc) return rc;
  if (p->priv) { rc = store_lz4_check(p->priv); if (rc) return rc; }   // a corrupt compressed buffer fails the execution
  return 0;
}
static int collect_partial_rows(sd_plan* p) {
  int rc = launch_what_is_pending(p);
  if (rc) return rc;
  if (p->finished_nrows >= 0) return 0;
  const int mode = p->spec.mode;
  rc = mode == MODE_HASH ? finish_hash(p) : mode == MODE_PROJECT ? finish_project(p) : finish_dense(p);
  if (rc) return rc;
  p->metrics[0] = p->finished_nrows;
  // the rows are host bytes, or device rows holding their own string bytes, and the stream has drained: the scan reads no
  // store memory any more (a cached plan sitting idle between queries pins nothing)
  p->pins.release();
  return 0;
}

int sd_plan_finish(sd_plan* p, void* out_rows, int64_t cap, int64_t* out_len, int64_t* out_nrows) {
  if (p && p->spec.mode == MODE_MUTATE) return set_error(SD_ERR_STATE, "sd_plan_finish: an UPDATE / DELETE plan keeps no result rows or partials");
  if (!p || !out_len) return set_error(SD_ERR_INVALID, "sd_plan_finish: null argument");
  int rc = collect_partial_rows(p);
  if (rc) return rc;
  if (p->dev_rows_len >= 0) {   // projected rows written by the GPU: one copy, straight into the caller's buffer
    *out_len = p->dev_rows_len;
    if (out_nrows) *out_nrows = p->finished_nrows;
    if (p->dev_rows_len > cap) return set_error(SD_ERR_OVERFLOW, "sd_plan_finish: output needs %lld bytes", (long long)p->dev_rows_len);
    if (p->dev_rows_len) SD_CUDA(cudaMemcpyAsync(out_rows, p->roww.d_rows, (size_t)p->dev_rows_len, cudaMemcpyDeviceToHost, p->stream));
    SD_CUDA(cudaStreamSynchronize(p->stream));
    return 0;
  }
  *out_len = (int64_t)p->finished_rows.size();
  if (out_nrows) *out_nrows = p->finished_nrows;
  if ((int64_t)p->finished_rows.size() > cap) return set_error(SD_ERR_OVERFLOW, "sd_plan_finish: output needs %zu bytes", p->finished_rows.size());
  if (!p->finished_rows.empty()) memcpy(out_rows, p->finished_rows.data(), p->finished_rows.size());
  return 0;
}

int sd_plan_reset(sd_plan* p) {
  if (!p) return set_error(SD_ERR_INVALID, "null plan");
  SD_CUDA(cudaSetDevice(p->device));
  SD_CUDA(cudaStreamSynchronize(p->stream));
  p->pins.release();
  p->pending.clear();
  p->pending_bytes = 0;
  p->result_init = false;
  p->hash_init = false;
  p->launch_log.clear();
  p->launch_records.clear();
  p->replay_kind = SDX_REPLAY_NONE;
  p->exec_batches.clear();
  p->finished_nrows = -1;
  p->dev_rows_len = -1;
  memset(p->rollup_info, 0, sizeof(p->rollup_info));
  if (p->d_out_count) SD_CUDA(cudaMemsetAsync(p->d_out_count, 0, 8, p->stream));
  p->have_timing = false;
  p->ev_used = 0;
  p->agg_ms = 0;
  SD_CUDA(cudaMemsetAsync(p->d_counters, 0, 64, p->stream));
  memset(p->metrics, 0, sizeof(p->metrics));
  p->scratch.reset();
  p->pinned.reset();
  if (p->priv) {
    cudaStreamSynchronize(p->priv->copy_stream);
    for (int k = 0; k + 1 < p->priv->num_copy_streams; k++) cudaStreamSynchronize(p->priv->extra_streams[k]);
    p->priv->batches.clear(); p->priv->arena.reset(); p->priv->version++; p->priv->h2d_bytes = 0;
    p->priv->pending_lz4.clear();
    store_lz4_check(p->priv);   // waits for queued expansions (their result is being discarded) and releases the staging
    p->priv->lz4_stage.reset();
  }
  // key dictionaries persist across executions of a cached plan only if the scan cache refers to them
  if (!p->cache.valid) {
    for (auto& m : p->key_ids) m.clear();
    for (auto& v : p->key_vals) v.clear();
    std::fill(p->key_null_id.begin(), p->key_null_id.end(), -1);
  }
  return 0;
}

int sd_plan_metrics(sd_plan* p, int64_t out[SD_NUM_METRICS]) {
  if (!p) return set_error(SD_ERR_INVALID, "null plan");
  memcpy(out, p->metrics, sizeof(p->metrics));
  return 0;
}

int sdx_plan_rollup_info(sd_plan* p, double out[4]) {
  if (!p || !out) return set_error(SD_ERR_INVALID, "sdx_plan_rollup_info: null argument");
  memcpy(out, p->rollup_info, sizeof(p->rollup_info));
  return 0;
}

int sdx_plan_launch_log(sd_plan* p, int64_t* out, int32_t cap, int32_t* n) {
  if (!p || !n || cap < 0 || (cap > 0 && !out)) return set_error(SD_ERR_INVALID, "sdx_plan_launch_log: bad arguments");
  const int32_t have = (int32_t)(p->launch_records.size() / SDX_LAUNCH_WORDS);
  *n = have;
  if (cap > 0) memcpy(out, p->launch_records.data(), (size_t)std::min(cap, have) * SDX_LAUNCH_WORDS * 8);
  if (cap < have) return set_error(SD_ERR_OVERFLOW, "sdx_plan_launch_log: %d records", have);
  return 0;
}

void sd_plan_destroy(sd_plan* p) {
  if (!p) return;
  cudaSetDevice(p->device);
  if (p->stream) cudaStreamSynchronize(p->stream);
  p->pins.release();   // (the registry outlives a store destroyed before this plan)
  if (p->own_stream && p->stream) cudaStreamDestroy(p->stream);
  if (p->ev_start) cudaEventDestroy(p->ev_start);
  if (p->ev_stop) cudaEventDestroy(p->ev_stop);
  for (auto& e : p->ev_pairs) { cudaEventDestroy(e.first); cudaEventDestroy(e.second); }
  if (p->d_state) cudaFree(p->d_state);
  if (p->h_pinned) cudaFreeHost(p->h_pinned);
  if (p->d_partials) cudaFree(p->d_partials);
  hash_free(p);
  table_free(p->rollup);
  if (p->d_rollup_meta) cudaFree(p->d_rollup_meta);
  if (p->ev_rollup[0]) { cudaEventDestroy(p->ev_rollup[0]); cudaEventDestroy(p->ev_rollup[1]); }
  if (p->d_out) cudaFree(p->d_out);
  if (p->h_recs) cudaFreeHost(p->h_recs);
  p->roww.release();
  if (p->d_out_count) cudaFree(p->d_out_count);
  if (p->d_hash_ident) cudaFree(p->d_hash_ident);
  if (p->d_ticket) cudaFree(p->d_ticket);
  if (p->d_litpool) cudaFree(p->d_litpool);
  if (p->priv) sd_store_destroy(p->priv);
  delete p;
}

// ---- dense partial table export/import for an on-device exchange (NCCL all-reduce) --------------
int sd_plan_partials_layout(sd_plan* p, int32_t* ngroups, int32_t* nslots, int32_t* slot_is_f64) {
  if (p && p->spec.mode == MODE_MUTATE) return set_error(SD_ERR_STATE, "sd_plan_partials_layout: an UPDATE / DELETE plan keeps no result rows or partials");
  if (!p) return set_error(SD_ERR_INVALID, "null plan");
  if (!p->spec.sets.empty()) return set_error(SD_ERR_UNSUPPORTED, "sd_plan_partials_layout: a grouping-sets plan has no dense partials");
  if (!p->spec.shifts.empty()) return set_error(SD_ERR_UNSUPPORTED, "sd_plan_partials_layout: shifted sums (moments, covariance) of different GPUs do not add");
  if (p->spec.norder > 0) return set_error(SD_ERR_UNSUPPORTED, "sd_plan_partials_layout: FIRST / LAST order keys of different GPUs do not compare");
  const int ns = (int)p->spec.slots.size();
  if (ngroups) *ngroups = p->ngroups;
  if (nslots) *nslots = ns;
  if (slot_is_f64) for (int s = 0; s < ns; s++) { const int op = p->spec.slots[s].op; slot_is_f64[s] = op == SLOT_ADD_F64 ? 1 : (op == SLOT_ADD_I64 ? 0 : -1); }
  return 0;
}
int sd_plan_export_partials(sd_plan* p, void* dev_out, int64_t cap_bytes) {
  if (p && p->spec.mode == MODE_MUTATE) return set_error(SD_ERR_STATE, "sd_plan_export_partials: an UPDATE / DELETE plan keeps no result rows or partials");
  if (!p || !dev_out) return set_error(SD_ERR_INVALID, "null argument");
  if (p->spec.mode == MODE_HASH || p->spec.mode == MODE_PROJECT) return set_error(SD_ERR_UNSUPPORTED, "dense partials exist only for no-key / dictionary-keyed plans");
  if (!p->spec.sets.empty()) return set_error(SD_ERR_UNSUPPORTED, "sd_plan_export_partials: a grouping-sets plan has no dense partials");
  if (!p->spec.shifts.empty()) return set_error(SD_ERR_UNSUPPORTED, "sd_plan_export_partials: shifted sums (moments, covariance) of different GPUs do not add");
  if (p->spec.norder > 0) return set_error(SD_ERR_UNSUPPORTED, "sd_plan_export_partials: FIRST / LAST order keys of different GPUs do not compare");
  SD_CUDA(cudaSetDevice(p->device));
  int rc = flush_pending(p);
  if (rc) return rc;
  if (!p->result_init) { rc = init_result(p, 1); if (rc) return rc; p->ngroups = 1; }
  const size_t bytes = (size_t)p->ngroups * p->spec.slots.size() * 8;
  if ((int64_t)bytes > cap_bytes) return set_error(SD_ERR_OVERFLOW, "export needs %zu bytes", bytes);
  SD_CUDA(cudaMemcpyAsync(dev_out, p->d_result, bytes, cudaMemcpyDeviceToDevice, p->stream));
  return 0;
}
int sd_plan_import_partials(sd_plan* p, const void* dev_in, int64_t bytes) {
  if (p && p->spec.mode == MODE_MUTATE) return set_error(SD_ERR_STATE, "sd_plan_import_partials: an UPDATE / DELETE plan keeps no result rows or partials");
  if (!p || !dev_in) return set_error(SD_ERR_INVALID, "null argument");
  if (p->spec.mode == MODE_HASH || p->spec.mode == MODE_PROJECT) return set_error(SD_ERR_UNSUPPORTED, "dense partials exist only for no-key / dictionary-keyed plans");
  if (!p->spec.sets.empty()) return set_error(SD_ERR_UNSUPPORTED, "sd_plan_import_partials: a grouping-sets plan has no dense partials");
  if (!p->spec.shifts.empty()) return set_error(SD_ERR_UNSUPPORTED, "sd_plan_import_partials: shifted sums (moments, covariance) of different GPUs do not add");
  if (p->spec.norder > 0) return set_error(SD_ERR_UNSUPPORTED, "sd_plan_import_partials: FIRST / LAST order keys of different GPUs do not compare");
  p->finished_nrows = -1;
  p->dev_rows_len = -1;
  SD_CUDA(cudaSetDevice(p->device));
  const size_t want = (size_t)p->ngroups * p->spec.slots.size() * 8;
  if ((size_t)bytes != want) return set_error(SD_ERR_INVALID, "import expects %zu bytes", want);
  SD_CUDA(cudaMemcpyAsync(p->d_result, dev_in, want, cudaMemcpyDeviceToDevice, p->stream));
  return 0;
}

// ---- row-buffer rows: the hybrid scan's first element (ColumnTableScan.scala:572-588) ----------------
// nrows UnsafeRows of the plan's scan columns -> one Uncompressed/Dictionary pseudo-batch.
int sd_rows_submit(sd_plan* p, const void* rows, int64_t len, int32_t nrows) {
  if (!p || (!rows && nrows > 0)) return set_error(SD_ERR_INVALID, "sd_rows_submit: null argument");
  if (nrows <= 0) return 0;
  const int nc = (int)p->spec.cols.size();
  std::vector<std::vector<uint8_t>> bufs(nc);
  std::vector<std::vector<HVal>> colv(nc, std::vector<HVal>((size_t)nrows));
  const uint8_t* r = reinterpret_cast<const uint8_t*>(rows);
  int64_t pos = 0;
  for (int i = 0; i < nrows; i++) {
    if (pos + 8 > len) return set_error(SD_ERR_INVALID, "sd_rows_submit: truncated row stream");
    int64_t sz;
    memcpy(&sz, r + pos, 8);
    if (sz < 0 || pos + 8 + sz > len) return set_error(SD_ERR_INVALID, "sd_rows_submit: bad row size");
    for (int c = 0; c < nc; c++)
      if (!unsafe_field(r + pos + 8, sz, nc, c, p->spec.cols[c].type, &colv[c][i])) return set_error(SD_ERR_INVALID, "sd_rows_submit: malformed UnsafeRow");
    pos += 8 + sz;
  }
  for (int c = 0; c < nc; c++) {
    const int t = p->spec.cols[c].type;
    std::vector<uint64_t> nw(((size_t)nrows + 63) / 64, 0);
    bool any_null = false;
    for (int i = 0; i < nrows; i++) if (colv[c][i].isnull) { nw[i >> 6] |= 1ull << (i & 63); any_null = true; }
    if (any_null && !p->spec.cols[c].nullable) return set_error(SD_ERR_INVALID, "NULL in NOT NULL column %d of the row buffer", c);
    while (!nw.empty() && nw.back() == 0) nw.pop_back();
    std::vector<uint8_t>& b = bufs[c];
    auto put32 = [&](int32_t v) { b.insert(b.end(), reinterpret_cast<uint8_t*>(&v), reinterpret_cast<uint8_t*>(&v) + 4); };
    if (t == SD_STRING) {   // first-seen dictionary
      std::unordered_map<std::string, int> ids;
      std::vector<std::string> vals;
      std::vector<int32_t> idx;
      for (int i = 0; i < nrows; i++) {
        if (colv[c][i].isnull) continue;
        auto it = ids.find(colv[c][i].s);
        if (it == ids.end()) { it = ids.emplace(colv[c][i].s, (int)vals.size()).first; vals.push_back(colv[c][i].s); }
        idx.push_back(it->second);
      }
      const bool big = vals.size() > 32767;
      put32(big ? ENC_BIG_DICTIONARY : ENC_DICTIONARY);
      put32((int32_t)nw.size() * 8);
      b.insert(b.end(), reinterpret_cast<uint8_t*>(nw.data()), reinterpret_cast<uint8_t*>(nw.data()) + nw.size() * 8);
      put32((int32_t)vals.size());
      for (auto& s : vals) { put32((int32_t)s.size()); b.insert(b.end(), s.begin(), s.end()); }
      for (int32_t x : idx) { if (big) put32(x); else { int16_t s16 = (int16_t)x; b.insert(b.end(), reinterpret_cast<uint8_t*>(&s16), reinterpret_cast<uint8_t*>(&s16) + 2); } }
    } else {
      put32(ENC_UNCOMPRESSED);
      put32((int32_t)nw.size() * 8);
      b.insert(b.end(), reinterpret_cast<uint8_t*>(nw.data()), reinterpret_cast<uint8_t*>(nw.data()) + nw.size() * 8);
      for (int i = 0; i < nrows; i++) {
        const HVal& v = colv[c][i];
        if (v.isnull) continue;
        switch (t) {
          case SD_BOOLEAN: case SD_BYTE: b.push_back((uint8_t)v.i); break;
          case SD_SHORT: { int16_t x = (int16_t)v.i; b.insert(b.end(), reinterpret_cast<uint8_t*>(&x), reinterpret_cast<uint8_t*>(&x) + 2); break; }
          case SD_INT: case SD_DATE: put32((int32_t)v.i); break;
          case SD_FLOAT: { float x = (float)v.d; b.insert(b.end(), reinterpret_cast<uint8_t*>(&x), reinterpret_cast<uint8_t*>(&x) + 4); break; }
          case SD_DOUBLE: { double x = v.d; b.insert(b.end(), reinterpret_cast<uint8_t*>(&x), reinterpret_cast<uint8_t*>(&x) + 8); break; }
          default: { int64_t x = v.i; b.insert(b.end(), reinterpret_cast<uint8_t*>(&x), reinterpret_cast<uint8_t*>(&x) + 8); break; }
        }
      }
    }
  }
  std::vector<const void*> ptrs(nc);
  std::vector<int64_t> lens(nc);
  for (int c = 0; c < nc; c++) { ptrs[c] = bufs[c].data(); lens[c] = (int64_t)bufs[c].size(); }
  sd_batch b;
  memset(&b, 0, sizeof(b));
  b.num_rows = nrows; b.ncols = nc; b.col_bufs = ptrs.data(); b.col_lens = lens.data(); b.bucket_id = -1; b.batch_id = -1;
  const int64_t seen_before = p->metrics[2];
  int rc = sd_batch_submit(p, &b);
  p->metrics[2] = seen_before;       // the row buffer is not a column batch
  if (!rc) p->metrics[1] += nrows;   // numRowsBuffer
  return rc;
}

// ---- merge of partial rows (host, sd_aggregate.cpp) ------------------------------------------------------
static int merge_to_caller(const PlanSpec& sp, const void* partial_rows, int64_t len, bool evaluate, void* out_rows, int64_t cap,
                           int64_t* out_len, int64_t* out_nrows) {
  if (!out_len) return set_error(SD_ERR_INVALID, "merge: null out_len");
  std::vector<uint8_t> out;
  std::string err;
  int rc = merge_rows(sp, partial_rows, len, evaluate, out, out_nrows, err);
  if (rc) return set_error(rc, "%s", err.c_str());
  *out_len = (int64_t)out.size();
  if ((int64_t)out.size() > cap) return set_error(SD_ERR_OVERFLOW, "merge: output needs %zu bytes", out.size());
  if (!out.empty()) memcpy(out_rows, out.data(), out.size());
  return 0;
}

int sd_final_merge(const sd_plan_desc* desc, const void* partial_rows, int64_t len, void* out_rows, int64_t cap,
                   int64_t* out_len, int64_t* out_nrows) {
  PlanSpec sp;
  std::string err;
  int rc = analyze_plan(desc, sp, err);
  if (rc) return set_error(rc, "sd_final_merge: %s", err.c_str());
  return merge_to_caller(sp, partial_rows, len, true, out_rows, cap, out_len, out_nrows);
}

/* same merge, reusing the analysis of an existing plan handle (no per-call plan analysis) */
int sd_plan_final_merge(sd_plan* p, const void* partial_rows, int64_t len, void* out_rows, int64_t cap,
                        int64_t* out_len, int64_t* out_nrows) {
  if (!p) return set_error(SD_ERR_INVALID, "null plan");
  return merge_to_caller(p->spec, partial_rows, len, true, out_rows, cap, out_len, out_nrows);
}

/* partial rows of several partitions -> one merged set of PARTIAL rows (same schema) */
int sd_partial_merge(const sd_plan_desc* desc, const void* partial_rows, int64_t len, void* out_rows, int64_t cap,
                     int64_t* out_len, int64_t* out_nrows) {
  PlanSpec sp;
  std::string err;
  int rc = analyze_plan(desc, sp, err);
  if (rc) return set_error(rc, "sd_partial_merge: %s", err.c_str());
  return merge_to_caller(sp, partial_rows, len, false, out_rows, cap, out_len, out_nrows);
}
int sd_plan_partial_merge(sd_plan* p, const void* partial_rows, int64_t len, void* out_rows, int64_t cap,
                          int64_t* out_len, int64_t* out_nrows) {
  if (!p) return set_error(SD_ERR_INVALID, "null plan");
  return merge_to_caller(p->spec, partial_rows, len, false, out_rows, cap, out_len, out_nrows);
}

// ---- the one exchange of the path (SURVEY.md 8e): every partition's partial rows -> all ranks, merged ----------
// Partial rows travel BY VALUE (keys as bytes, like the reference's shuffle of UnsafeRows between the partial and the
// final HashAggregate, SnappyStrategies.scala:566-604): dictionary ids are private to a partition.  One ncclAllGather
// of a fixed-capacity blob per rank [magic:4][flags:4][len:8][rows]; a rank whose rows do not fit says so in its header,
// every rank sees every header, so all of them grow the capacity and repeat in lock step (the capacity sticks).
struct sd_comm {
  void* nccl = nullptr;
  int rank = 0, world = 1, device = 0;
  size_t cap = 2048;               // bytes per rank, header included
  uint8_t *d_send = nullptr, *d_recv = nullptr, *h_send = nullptr, *h_recv = nullptr;
  size_t alloc_cap = 0;
  int64_t exchanges = 0, regrows = 0;
};
static int comm_buffers(sd_comm* c) {
  if (c->alloc_cap >= c->cap) return 0;
  if (c->d_send) { cudaFree(c->d_send); cudaFree(c->d_recv); cudaFreeHost(c->h_send); cudaFreeHost(c->h_recv); c->d_send = c->d_recv = c->h_send = c->h_recv = nullptr; }
  SD_CUDA(cudaMalloc(&c->d_send, c->cap));
  SD_CUDA(cudaMalloc(&c->d_recv, c->cap * (size_t)c->world));
  SD_CUDA(cudaMallocHost(&c->h_send, c->cap));
  SD_CUDA(cudaMallocHost(&c->h_recv, c->cap * (size_t)c->world));
  c->alloc_cap = c->cap;
  return 0;
}
constexpr uint32_t COMM_MAGIC = 0x53445831u;   // "SDX1"

int sd_comm_unique_id(void* out_id) {
  if (!out_id) return set_error(SD_ERR_INVALID, "sd_comm_unique_id: null argument");
  return comm_unique_id(out_id);
}
int sd_comm_create(const void* id, int32_t rank, int32_t world, int32_t device, sd_comm** out) {
  if (!id || !out || world < 1 || rank < 0 || rank >= world) return set_error(SD_ERR_INVALID, "sd_comm_create: bad arguments");
  SD_CUDA(cudaSetDevice(device));
  std::unique_ptr<sd_comm> c(new sd_comm());
  c->rank = rank; c->world = world; c->device = device;
  int rc = comm_init(id, rank, world, &c->nccl);
  if (rc) return rc;
  *out = c.release();
  return 0;
}
void sd_comm_destroy(sd_comm* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  comm_destroy(c->nccl);
  if (c->d_send) { cudaFree(c->d_send); cudaFree(c->d_recv); cudaFreeHost(c->h_send); cudaFreeHost(c->h_recv); }
  delete c;
}
int sd_comm_info(sd_comm* c, int64_t out[4]) {
  if (!c || !out) return set_error(SD_ERR_INVALID, "null argument");
  out[0] = c->world; out[1] = (int64_t)c->cap; out[2] = c->exchanges; out[3] = c->regrows;
  return 0;
}

// The exchange's blob of one rank: [magic u32][flags u32][len u64][payload].  flags bit 0: the payload did not fit the slot (only
// the header travelled; every rank doubles the slot and repeats).  flags bit 1: DENSE form -- the payload is this rank's key
// dictionaries followed by the raw [counters][ngroups x slots] state exactly as the kernel left it in HBM:
//   [ngroups i32][nk i32][radix i32 x nk][null id i32 x nk] { [n u32] { [len u32][bytes] } x n } x nk  pad to 8  [state u64 x (8 + ngroups*ns)]
// The sender queues header H2D + a device-to-device copy of the state + the all-gather behind its scan kernel and meets the
// result with ONE synchronisation: no read-back of its own state, no row building, no second upload before the collective
// (the by-value form below needs all three).  Receivers turn each rank's state into partial rows with that rank's dictionaries.
// averaged host-side laps of the per-query path (SD_DEBUG_TIMING=1; printed every 64 calls)
struct LapStats {
  static constexpr int N = 8;
  double sum[N] = {0}; int64_t calls = 0; const char* names[N] = {nullptr};
  std::chrono::steady_clock::time_point t0;
  bool on = getenv("SD_DEBUG_TIMING") != nullptr;
  void begin() { if (on) t0 = std::chrono::steady_clock::now(); }
  void lap(int i, const char* name) {
    if (!on) return;
    const auto t = std::chrono::steady_clock::now();
    sum[i] += std::chrono::duration<double, std::micro>(t - t0).count(); names[i] = name; t0 = t;
  }
  void end(const char* what, int rank) {
    if (!on || (++calls % 64) != 0) return;
    fprintf(stderr, "[%s rank %d] avg us over %lld calls:", what, rank, (long long)calls);
    for (int i = 0; i < N; i++) if (names[i]) fprintf(stderr, "  %s %.1f", names[i], sum[i] / (double)calls);
    fprintf(stderr, "\n");
  }
};
static bool dense_exchange_eligible(const sd_plan* p) {
  if (getenv("SD_TUNE_EXCHANGE_ROWS")) return false;
  const PlanSpec& sp = p->spec;
  if (sp.mode != MODE_NOKEY && sp.mode != MODE_GROUPS) return false;
  if (p->finished_nrows >= 0) return false;   // rows already materialised by an earlier call
  if (!sp.sets.empty()) return false;         // the ranks' rolled-up rows are gathered and merged by (keys, gid)
  // record addresses point into this rank's HBM; limb sums are exact below 2^31 rows of ONE execution, and summing them over
  // the ranks could pass 2^64, so wide-DECIMAL sums take the by-value exchange, whose merge adds recombined 128-bit totals with
  // an overflow check
  for (const auto& m : sp.agg_map) if (m.hold == HOLD_REF || m.hold == HOLD_LIMBS) return false;
  return true;
}

int sd_plan_exchange(sd_plan* p, sd_comm* c) {
  if (p && p->spec.mode == MODE_MUTATE) return set_error(SD_ERR_STATE, "sd_plan_exchange: an UPDATE / DELETE plan keeps no result rows or partials");
  if (!p || !c) return set_error(SD_ERR_INVALID, "sd_plan_exchange: null argument");
  if (c->device != p->device) return set_error(SD_ERR_INVALID, "communicator lives on device %d, plan on %d", c->device, p->device);
  static thread_local LapStats laps;
  laps.begin();
  int rc = launch_what_is_pending(p);
  if (rc) return rc;
  const PlanSpec& sp = p->spec;
  const int ns = (int)sp.slots.size(), nk = (int)sp.keys.size();
  const bool dense = dense_exchange_eligible(p);
  std::vector<uint8_t> dense_hdr;
  size_t state_bytes = 0;
  if (dense) {
    if (!p->result_init) { rc = init_result(p, 1); if (rc) return rc; p->ngroups = 1; }
    const size_t ne = (size_t)p->ngroups * ns;
    rc = ensure_result(p, ne);
    if (rc) return rc;
    state_bytes = (STATE_HDR + result_words(sp, p->ngroups)) * 8;   // moment aggregates: this rank's K words travel with it
    auto put32 = [&](uint32_t v) { const uint8_t* q = reinterpret_cast<const uint8_t*>(&v); dense_hdr.insert(dense_hdr.end(), q, q + 4); };
    put32((uint32_t)p->ngroups); put32((uint32_t)nk);
    for (int k = 0; k < nk; k++) put32((uint32_t)p->radix[k]);
    for (int k = 0; k < nk; k++) put32((uint32_t)p->key_null_id[k]);
    for (int k = 0; k < nk; k++) {
      put32((uint32_t)p->key_vals[k].size());
      for (const std::string& v : p->key_vals[k]) { put32((uint32_t)v.size()); dense_hdr.insert(dense_hdr.end(), v.begin(), v.end()); }
    }
    dense_hdr.resize((dense_hdr.size() + 7) & ~size_t(7), 0);
  } else {
    rc = collect_partial_rows(p);
    if (rc) return rc;
    rc = rows_to_host(p);
    if (rc) return rc;
  }
  const std::vector<uint8_t>& mine = p->finished_rows;
  for (;;) {
    rc = comm_buffers(c);
    if (rc) return rc;
    const size_t room = c->cap - 16, n = dense ? dense_hdr.size() + state_bytes : mine.size();
    const bool fits = n <= room;
    const uint32_t hdr32[2] = {COMM_MAGIC, (fits ? 0u : 1u) | (dense ? 2u : 0u)};
    const uint64_t len64 = n;
    memcpy(c->h_send, hdr32, 8);
    memcpy(c->h_send + 8, &len64, 8);
    if (dense) {
      if (fits) {
        memcpy(c->h_send + 16, dense_hdr.data(), dense_hdr.size());
        SD_CUDA(cudaMemcpyAsync(c->d_send, c->h_send, 16 + dense_hdr.size(), cudaMemcpyHostToDevice, p->stream));
        SD_CUDA(cudaMemcpyAsync(c->d_send + 16 + dense_hdr.size(), p->d_state, state_bytes, cudaMemcpyDeviceToDevice, p->stream));
      } else {
        SD_CUDA(cudaMemcpyAsync(c->d_send, c->h_send, 16, cudaMemcpyHostToDevice, p->stream));
      }
    } else {
      const size_t sent = std::min(n, room);
      if (sent) memcpy(c->h_send + 16, mine.data(), sent);
      SD_CUDA(cudaMemcpyAsync(c->d_send, c->h_send, 16 + sent, cudaMemcpyHostToDevice, p->stream));
    }
    laps.lap(0, "prepare+copies");
    rc = comm_all_gather_bytes(c->nccl, c->d_send, c->d_recv, c->cap, p->stream);
    if (rc) return rc;
    SD_CUDA(cudaMemcpyAsync(c->h_recv, c->d_recv, c->cap * (size_t)c->world, cudaMemcpyDeviceToHost, p->stream));
    laps.lap(1, "enqueue-allgather");
    SD_CUDA(cudaStreamSynchronize(p->stream));
    laps.lap(2, "wait(kernel+allgather+d2h)");
    c->exchanges++;
    size_t maxlen = 0;
    for (int r = 0; r < c->world; r++) {
      const uint8_t* h = c->h_recv + (size_t)r * c->cap;
      uint32_t magic; uint64_t l;
      memcpy(&magic, h, 4); memcpy(&l, h + 8, 8);
      if (magic != COMM_MAGIC) return set_error(SD_ERR_CUDA, "sd_plan_exchange: bad header from rank %d", r);
      maxlen = std::max<size_t>(maxlen, (size_t)l);
    }
    if (maxlen <= room) break;
    size_t ncap = c->cap;
    while (ncap - 16 < maxlen) ncap *= 2;
    c->cap = ncap;   // every rank computes the same value from the same headers
    c->regrows++;
  }
  std::vector<uint8_t> all;
  for (int r = 0; r < c->world; r++) {
    const uint8_t* h = c->h_recv + (size_t)r * c->cap;
    uint32_t flags; uint64_t l;
    memcpy(&flags, h + 4, 4); memcpy(&l, h + 8, 8);
    const uint8_t* q = h + 16;
    const uint8_t* const end = q + l;
    if (!(flags & 2u)) { all.insert(all.end(), q, end); continue; }
    // dense form: that rank's dictionaries, then its state
    auto get32 = [&](uint32_t* v) { if (q + 4 > end) return false; memcpy(v, q, 4); q += 4; return true; };
    auto bad = [&]() { return set_error(SD_ERR_CUDA, "sd_plan_exchange: malformed dense blob from rank %d", r); };
    uint32_t ng = 0, rnk = 0;
    if (!get32(&ng) || !get32(&rnk) || (int)rnk != nk || ng == 0) return bad();
    int32_t radix[MAX_KEYS] = {1, 1, 1, 1};
    std::vector<int> null_id((size_t)nk, -1);
    std::vector<std::vector<std::string>> vals((size_t)nk);
    uint64_t prod = 1;
    for (int k = 0; k < nk; k++) { uint32_t v; if (!get32(&v) || v == 0) return bad(); radix[k] = (int32_t)v; prod *= v; }
    if (prod != ng) return bad();
    for (int k = 0; k < nk; k++) { uint32_t v; if (!get32(&v)) return bad(); null_id[(size_t)k] = (int32_t)v; }
    for (int k = 0; k < nk; k++) {
      uint32_t nv; if (!get32(&nv)) return bad();
      for (uint32_t i = 0; i < nv; i++) {
        uint32_t sl; if (!get32(&sl) || q + sl > end) return bad();
        vals[(size_t)k].emplace_back(reinterpret_cast<const char*>(q), sl); q += sl;
      }
      // (a radix may exceed the dictionary by the NULL id; an id beyond both never has rows)
      if ((size_t)radix[k] > vals[(size_t)k].size()) vals[(size_t)k].resize((size_t)radix[k]);
    }
    q = h + 16 + (((size_t)(q - (h + 16)) + 7) & ~size_t(7));
    if (q + (STATE_HDR + result_words(sp, (int)ng)) * 8 != end) return bad();
    std::vector<uint64_t> st(STATE_HDR + result_words(sp, (int)ng));
    memcpy(st.data(), q, st.size() * 8);
    const int64_t nr = dense_rows_from_state(sp, st.data() + STATE_HDR, (int)ng, radix, null_id, vals, nullptr, all);
    if (r == c->rank) {   // this rank's own execution metrics come back with its blob
      update_agg_time(p);
      p->metrics[6] = (int64_t)(p->agg_ms * 1e6);
      p->metrics[8] = (int64_t)st[0];
      p->metrics[11] = (int64_t)st[0];
      p->metrics[0] = nr;
    }
  }
  laps.lap(3, "decode-blobs");
  std::vector<uint8_t> merged;
  int64_t nrows = 0;
  std::string err;
  rc = merge_rows(p->spec, all.data(), (int64_t)all.size(), false, merged, &nrows, err);
  if (rc) return set_error(rc, "%s", err.c_str());
  p->finished_rows.swap(merged);
  p->finished_nrows = nrows;
  p->dev_rows_len = -1;
  laps.lap(4, "merge");
  laps.end("sd_plan_exchange", c->rank);
  return 0;
}

// one execution of a cached plan over a resident store, in one call: reset -> literals -> scan -> [exchange] ->
// partial rows (merged over all ranks when `comm` is given).  What a re-executed cached plan does per query in the
// reference (SnappySession plan cache: new literal values, same generated code).
int sd_plan_execute_store(sd_plan* p, sd_store* s, const int32_t* bucket_ids, int32_t nbuckets, const sd_literal* lits, int32_t nlits,
                          sd_comm* comm, void* out_rows, int64_t cap, int64_t* out_len, int64_t* out_nrows) {
  static thread_local LapStats laps;
  laps.begin();
  int rc = sd_plan_reset(p);
  if (rc) return rc;
  laps.lap(0, "reset");
  if (lits || nlits) { rc = sd_plan_set_literals(p, lits, nlits); if (rc) return rc; }
  rc = sd_plan_scan_store(p, s, bucket_ids, nbuckets);
  if (rc) return rc;
  laps.lap(1, "literals+scan-enqueue");
  if (comm) { rc = sd_plan_exchange(p, comm); if (rc) return rc; }
  laps.lap(2, "exchange");
  rc = sd_plan_finish(p, out_rows, cap, out_len, out_nrows);
  laps.lap(3, "finish");
  laps.end("sd_plan_execute_store", comm ? comm->rank : 0);
  return rc;
}

}  // extern "C"
