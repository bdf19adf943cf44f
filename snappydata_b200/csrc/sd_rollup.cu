// sd_rollup.cu -- GROUP BY ... WITH ROLLUP / CUBE / GROUPING SETS: the fine groups of one execution's plain GROUP BY k1..kn
// scan, rolled up into every grouping set at once.
//
// Spark plans these queries as Expand (every row once per set, absent keys NULL, spark_grouping_id appended) under the partial
// aggregate.  Every set is a coarsening of the grouping by all n keys and every slot of the scan is decomposable (slot_atomic
// combines it; moment and covariance sums are re-centred on the coarse group's shift; a FIRST / LAST pair keeps the fine group
// whose order key wins), so the device scans once with the plan's
// plain kernel and this kernel combines each (fine group, set) into a hash table keyed by (k1..kn with absent keys NULL, gid):
// work proportional to groups x sets, not to rows.
#include <algorithm>

#include "sd_host.h"
#include "sd_kernels.cuh"

namespace sd {

namespace {

// one thread per (fine group, set)
__global__ void rollup_kernel(RollupArgs a) {
  const uint64_t total = (uint64_t)a.nfine * (uint64_t)a.nsets;
  const int nk = a.nk;
  for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < total; w += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t e = (uint32_t)(w / (uint64_t)a.nsets);
    const int set = (int)(w % (uint64_t)a.nsets);
    const uint64_t* sv = a.vals + (size_t)e * a.ns;
    if (a.rows_slot >= 0 && sv[a.rows_slot] == 0ull) continue;   // dense table: a key combination no row had
    int64_t kc[MAX_HASH_KEYS];
    uint32_t knull = 0;
    if (a.keys) {   // compacted hash entries
      for (int k = 0; k < nk; k++) kc[k] = a.keys[(size_t)e * nk + k];
      knull = a.knull[e];
    } else {        // dense table: the mixed-radix index -> query-global dictionary ids
      uint32_t rem = e;
      for (int k = nk - 1; k >= 0; k--) {
        const int id = (int)(rem % (uint32_t)a.radix[k]);
        rem /= (uint32_t)a.radix[k];
        kc[k] = id;
        if (id == a.null_id[k]) { kc[k] = 0; knull |= 1u << k; }
      }
    }
    const uint32_t mask = a.masks[set];
    for (int k = 0; k < nk; k++)
      if ((mask >> (nk - 1 - k)) & 1u) { kc[k] = 0; knull |= 1u << k; }   // absent from the set: NULL (SnappyParser's bit order)
    kc[nk] = (int64_t)mask;
    const int64_t c = hash_probe(a.out, kc, knull, nk + 1, a.strmask);
    if (c < 0) continue;   // the table overflowed: the host grows it and runs the roll-up again
    uint64_t* cv = a.out.vals + (size_t)c * a.ns;
    // moment / covariance sums: Sigma (x - K)^j of the fine group, re-centred on the coarse group's K' (the first fine K that
    // reaches it).  With d = K - K': S'_j = sum_i C(j, i) S_i d^(j-i), S_0 = n; S'_xy = S_xy + dy S_x + dx S_y + n dx dy
    double dsh[ROLLUP_MAX_SHIFTS];
    bool have[ROLLUP_MAX_SHIFTS];
    for (int i = 0; i < a.nsh; i++) {
      const uint64_t K = a.shifts[(size_t)e * a.nsh + i];
      have[i] = K != SHIFT_EMPTY;
      dsh[i] = 0.0;
      if (!have[i]) continue;   // no input in this fine group: its sums are 0
      dsh[i] = u2f(K) - u2f(shift_claim(a.out.shifts + (size_t)c * a.nsh + i, K));
    }
    for (int s = 0; s < a.ns; s++) {
      const int role = a.slot_role[s];
      uint64_t v = sv[s];
      if (role >= 0) {   // S_j of shift (role >> 3), j = role & 7
        const int i = role >> 3, j = role & 7;
        if (!have[i]) continue;
        const double d = dsh[i];
        double acc = 0.0, dp = 1.0;
        // binomial sum from the highest power down: C(j, j - m) S_{j - m} d^m
        double binom = 1.0;
        for (int m = 0; m <= j; m++) {
          const int q = j - m;
          const double Sq = q == 0 ? (double)sv[a.shift_count[i]] : u2f(sv[a.shift_pow[i * 4 + q - 1]]);
          acc += binom * Sq * dp;
          dp *= d;
          binom = binom * (double)(j - m) / (double)(m + 1);
        }
        v = f2u(acc);
      } else if (role <= -2) {   // S_xy of pair (-role - 2)
        const int q = -role - 2, ix = a.pair_x[q], iy = a.pair_y[q];
        if (!have[ix] || !have[iy]) continue;
        const double dx = dsh[ix], dy = dsh[iy];
        const double n = (double)sv[a.shift_count[ix]], Sx = u2f(sv[a.shift_pow[ix * 4]]), Sy = u2f(sv[a.shift_pow[iy * 4]]);
        v = f2u(u2f(v) + dy * Sx + dx * Sy + n * dx * dy);
      }
      const int op = a.slot_op[s];
      if (is_order_op(op)) { order_atomic<false>(op, cv + s, v, sv[s + 1]); s++; continue; }   // FIRST / LAST: the fine group's pair
      slot_atomic(op, cv + s, v);
    }
  }
}

}  // namespace

int rollup_launch(cudaStream_t stream, const RollupArgs& a) {
  const uint64_t total = (uint64_t)a.nfine * (uint64_t)a.nsets;
  if (total == 0) return 0;
  const int blocks = (int)std::min<uint64_t>(132 * 16, (total + 255) / 256);
  rollup_kernel<<<blocks, 256, 0, stream>>>(a);
  SD_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace sd
