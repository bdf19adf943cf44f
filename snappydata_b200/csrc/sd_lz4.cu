// sd_lz4.cu -- on-device LZ4 block decompression of stored column buffers (SURVEY.md 8f N1).
//
// The reference stores a column value as [-codecId:int32][uncompressedLen:int32][LZ4 block] when it is
// >= 2048 bytes and shrinks to <= 75 % (encoders/.../store/CompressionUtils.scala:53-61,102-110) and
// decompresses it on the CPU whenever a scan needs it (ColumnFormatEntry.scala:498-570,
// ColumnBatchIterator.scala:102-113).  Here only the COMPRESSED bytes cross PCIe; the block is expanded in
// HBM by one warp per buffer, many buffers per launch, launches of successive flushes overlapping each other.  The host decodes just the first bytes it needs to
// lay the buffer out (8-byte header, null words, dictionary) with the small prefix decoder below.
//
// LZ4 block format: sequences of [token][literal length ext*][literals][offset:2][match length ext*];
// token = (literal length << 4) | (match length - 4); the last sequence ends after its literals.
#include <cstdlib>
#include <cstring>
#include <vector>

#include "sd_host.h"

namespace sd {

// ---- host: decode at most `want` leading bytes of an LZ4 block (returns bytes produced, -1 if corrupt) --
int64_t lz4_decode_prefix(const uint8_t* src, int64_t src_len, uint8_t* dst, int64_t want) {
  int64_t s = 0, o = 0;
  while (s < src_len && o < want) {
    const uint8_t token = src[s++];
    int64_t lit = token >> 4;
    if (lit == 15) { uint8_t b; do { if (s >= src_len) return -1; b = src[s++]; lit += b; } while (b == 255); }
    if (s + lit > src_len) return -1;
    const int64_t lcopy = lit < want - o ? lit : want - o;
    memcpy(dst + o, src + s, (size_t)lcopy);
    o += lcopy; s += lit;
    if (o >= want || s >= src_len) break;
    if (s + 2 > src_len) return -1;
    const int64_t off = src[s] | ((int64_t)src[s + 1] << 8);
    s += 2;
    int64_t ml = (token & 15);
    if (ml == 15) { uint8_t b; do { if (s >= src_len) return -1; b = src[s++]; ml += b; } while (b == 255); }
    ml += 4;
    if (off == 0 || off > o) return -1;
    for (int64_t i = 0; i < ml && o < want; i++, o++) dst[o] = dst[o - off];
  }
  return o;
}

// ---- host: Snappy raw format (the reference's other codec, CompressionCodecId.SNAPPY_ID = 2, CompressionUtils.scala:125-168).
// preamble = uncompressed length as a varint; elements: tag & 3 = 0 literal (len-1 in the upper 6 bits, 60..63 = that
// many + 1 - 60 extra length bytes), 1 copy (len 4..11, 11-bit offset), 2 copy (len 1..64, 16-bit offset), 3 copy (32-bit offset).
int64_t snappy_decode(const uint8_t* src, int64_t n, uint8_t* dst, int64_t cap) {
  int64_t s = 0, ulen = 0;
  int shift = 0;
  for (;;) {
    if (s >= n || shift > 35) return -1;
    const uint8_t b = src[s++];
    ulen |= (int64_t)(b & 0x7f) << shift;
    if (!(b & 0x80)) break;
    shift += 7;
  }
  if (ulen > cap) return -1;
  int64_t o = 0;
  while (s < n) {
    const uint8_t tag = src[s++];
    int64_t len, off;
    switch (tag & 3) {
      case 0: {
        len = (tag >> 2) + 1;
        if (len > 60) {
          const int extra = (int)len - 60;
          if (s + extra > n) return -1;
          len = 0;
          for (int i = 0; i < extra; i++) len |= (int64_t)src[s + i] << (8 * i);
          len += 1;
          s += extra;
        }
        if (s + len > n || o + len > ulen) return -1;
        memcpy(dst + o, src + s, (size_t)len);
        s += len; o += len;
        continue;
      }
      case 1: if (s + 1 > n) return -1; len = 4 + ((tag >> 2) & 7); off = ((int64_t)(tag >> 5) << 8) | src[s]; s += 1; break;
      case 2: if (s + 2 > n) return -1; len = (tag >> 2) + 1; off = src[s] | ((int64_t)src[s + 1] << 8); s += 2; break;
      default: if (s + 4 > n) return -1; len = (tag >> 2) + 1; off = src[s] | ((int64_t)src[s + 1] << 8) | ((int64_t)src[s + 2] << 16) | ((int64_t)src[s + 3] << 24); s += 4; break;
    }
    if (off == 0 || off > o || o + len > ulen) return -1;
    for (int64_t i = 0; i < len; i++, o++) dst[o] = dst[o - off];
  }
  return o == ulen ? o : -1;
}

int decompress_envelope_host(const uint8_t* buf, int64_t len, std::vector<uint8_t>& out) {
  if (len < 8) return set_error(SD_ERR_INVALID, "compressed buffer shorter than its envelope");
  int32_t codec, ulen;
  memcpy(&codec, buf, 4); memcpy(&ulen, buf + 4, 4);
  codec = -codec;
  if (ulen < 0) return set_error(SD_ERR_INVALID, "compressed buffer: bad uncompressed length %d", ulen);
  out.assign((size_t)ulen + 16, 0);
  int64_t got = -1;
  if (codec == 1) got = lz4_decode_prefix(buf + 8, len - 8, out.data(), ulen);
  else if (codec == 2) got = snappy_decode(buf + 8, len - 8, out.data(), ulen);
  else return set_error(SD_ERR_UNSUPPORTED, "compressed buffer with unknown codec id %d (LZ4 = 1, Snappy = 2)", codec);
  if (got != ulen) return set_error(SD_ERR_INVALID, "corrupt %s payload (%lld of %d bytes)", codec == 1 ? "LZ4" : "Snappy", (long long)got, ulen);
  out.resize((size_t)ulen);
  return 0;
}

// ---- device: one warp per buffer, 32 sequences at a time -------------------------------------------------
// A column buffer is ONE LZ4 block (the reference compresses the whole value, CompressionUtils.scala:102-110), so
// the unit of independent work is the buffer and the time of a launch is the serial chain of its longest buffer.
// The first decoder here walked that chain one sequence at a time with every match source read coming back from
// L2: ~1200 cycles per sequence.  This one shortens
// the chain instead of adding warps:
//   * phase A: all lanes parse the token stream redundantly (warp-uniform loads) and lane i keeps sequence i of a
//     group of up to 32 -- the chain per sequence is one cached byte load, the copies are no longer part of it;
//   * phase B: lane i copies its own sequence.  Literals have no hazards.  A match may read bytes produced by an
//     earlier sequence of the same group, so matches run in rounds: a lane goes when its source range lies below
//     the output position of the first sequence that is still pending (that lane always qualifies);
//   * the most recent CFG::WIN bytes of output live in a shared-memory ring, so a round costs shared-memory
//     latency, not L2 latency; the ring is written out with coalesced 16-byte stores after every group.  Sources
//     farther back than the ring are read from HBM/L2 (they were flushed long before);
//   * sequences with long literal runs or long matches end the group and are copied by the whole warp;
//   * the parse is the serial part, so it is kept lean: while a whole group's worth of input and output remains,
//     the input is staged in a small shared-memory ring (coalesced 16-byte loads) and a short sequence -- at most
//     one length-extension byte each -- is parsed without per-field bounds checks (only the offset is validated);
//     anything else takes the fully checked path that reads HBM.  (The first version of this kernel spent ~110
//     instructions per sequence in the parse, most of its time.)
// Positions below are "shifted": P = output offset + (dst & 15), so that dst_al = dst - (dst & 15) is 16-byte
// aligned, byte P lives at dst_al[P] and in ring slot P & (CFG::WIN - 1), and ring vectors line up with HBM vectors.
constexpr int LZ_MAX_LIT = 32;         // longer literal runs / matches are copied by the whole warp
constexpr int LZ_MAX_ML = 64;
constexpr int LZ_SEQ_IN_MAX = 1 + 1 + LZ_MAX_LIT + 2 + 1;   // input bytes of a short sequence: token, <= 1 length byte each
constexpr uint32_t LZ_GROUP_IN = 32 * LZ_SEQ_IN_MAX + 16;   // input a group of short sequences can consume (+ slack)
constexpr uint32_t LZ_GROUP_OUT = 32 * (LZ_MAX_LIT + LZ_MAX_ML);

// Shape of the kernel: warps (= buffers) per CTA, output ring, input ring, piece size of whole-warp copies.
template <int WARPS_, int WIN_, int IN_, int PIECE_>
struct LzCfg {
  static constexpr int WARPS = WARPS_;
  static constexpr int WIN = WIN_;         // output ring bytes per warp (power of two)
  static constexpr int IN = IN_;           // ring of staged input bytes per warp (power of two)
  static constexpr int PIECE = PIECE_;     // whole-warp copies proceed in pieces of this size
  static constexpr uint32_t M = WIN_ - 1, IM = IN_ - 1;
  static constexpr size_t SMEM = (size_t)(WIN_ + IN_) * WARPS_;
  // the output ring must hold a piece being flushed, the piece (or group) being written and the flush's 16-byte slack;
  // the input ring a group's input plus the 512-byte staging step
  static_assert((WIN_ & (WIN_ - 1)) == 0 && (IN_ & (IN_ - 1)) == 0, "rings are powers of two");
  static_assert(2 * PIECE_ + LZ_GROUP_OUT + 16 <= WIN_ && 2 * LZ_GROUP_OUT + 16 <= WIN_, "output ring too small");
  static_assert(LZ_GROUP_IN + 512 <= IN_, "input ring too small");
};
// LzDefault is the original shape (4 warps per CTA).
// LzDense trades ring size for residency: the launch is a latency chain per buffer, so the aggregate expansion rate is
// (resident buffers) x (bytes per chain-time); with 1 warp and 10 KB per CTA 20 buffers fit an SM instead of 8.  It is
// selected with SD_TUNE_LZ4_DENSE=1; it passes the GPU parity tests (byte-exact against liblz4) but has not been TIMED
// yet (the round's GPU budget ended first); its ring invariants are also checked by tools/lz4_model.py.
typedef LzCfg<4, 16384, 4096, 4096> LzDefault;
typedef LzCfg<1, 8192, 2048, 2048> LzDense;

// ---- window parse (kernel template parameter PARSE == 1; opt-in with SD_TUNE_LZ4_PARSE=1) ------------------------
// The serial parse costs one dependent shared-memory round trip plus ~35 instructions per sequence.  The window parse
// examines LZ_WP input bytes per step without a chain: every position is parsed speculatively as if a token started
// there (`next token` per position, STOP where the checked path is needed), two doubling passes turn that into a 4-step
// jump, the chain from the window's first byte is walked four sequences at a time (8 dependent steps for 32 sequences)
// and each lane fills in its own member and extracts its fields; output positions come from a warp prefix sum.
// tools/lz4_model.py (window_parse) is the executable model of exactly this and cross-checks it against the serial
// parse; the kernel code below compiles but was written after the round's GPU budget ended: NOT yet run on hardware.
constexpr int LZ_WP = 256;
constexpr uint32_t LZ_STOP = 0xFFFFu;
static_assert(LZ_WP + LZ_SEQ_IN_MAX + 2 <= (int)LZ_GROUP_IN, "the window's speculative reads stay inside the staged input");

// parse the short sequence that would start at window position p (input byte s0 + p); returns the position of the
// next token (may lie beyond the window) or LZ_STOP when the sequence needs the checked path
template <class CFG>
__device__ __forceinline__ uint32_t lz_spec(const uint8_t* in, uint32_t s0, uint32_t p, uint32_t& lit_src, uint32_t& lit, uint32_t& q_off, uint32_t& ml) {
  const uint32_t token = in[(s0 + p) & CFG::IM];
  uint32_t q = p + 1;
  lit = token >> 4;
  ml = token & 15;
  bool ok = true;
  if (lit == 15) { const uint32_t e = in[(s0 + q) & CFG::IM]; q++; lit += e; ok = e != 255; }
  ok = ok && lit <= (uint32_t)LZ_MAX_LIT;
  if (!ok) lit = 0;   // keeps the speculative reads below inside the staged range
  lit_src = q;
  q += lit;
  q_off = q;
  q += 2;
  if (ml == 15) { const uint32_t e = in[(s0 + q) & CFG::IM]; q++; ml += e; ok = ok && e != 255; }
  ml += 4;
  ok = ok && ml <= (uint32_t)LZ_MAX_ML;
  return ok ? q : LZ_STOP;
}

// write ring bytes [flushed, floor16(upto)) to HBM; only the very first flush can start unaligned (the head)
template <class CFG>
__device__ __forceinline__ void lz_flush(const uint8_t* win, uint8_t* dst_al, uint32_t& flushed, uint32_t upto, int lane) {
  const uint32_t lim = upto & ~15u;
  if (lim <= flushed) return;
  if (flushed & 15u) {
    const uint32_t head_end = (flushed + 15u) & ~15u;
    for (uint32_t P = flushed + lane; P < head_end; P += 32) dst_al[P] = win[P & CFG::M];
    flushed = head_end;
  }
  const uint4* w = reinterpret_cast<const uint4*>(win);
  uint4* d = reinterpret_cast<uint4*>(dst_al);
  for (uint32_t v = (flushed >> 4) + lane; v < (lim >> 4); v += 32) d[v] = w[v & (CFG::WIN / 16 - 1)];
  flushed = lim;
}

// one lane copies its own match of <= LZ_MAX_ML bytes into the ring
template <class CFG>
__device__ __forceinline__ void lz_lane_match(uint8_t* win, const uint8_t* dst_al, uint32_t mdst, uint32_t msrc, uint32_t ml, uint32_t off, bool near) {
  uint32_t q = 0;
  if (off >= 8) {   // 8 source bytes never overlap the 8 bytes they produce: fetch them all, then store
    for (; q + 8 <= ml; q += 8) {
      uint8_t t[8];
      if (near) {
#pragma unroll
        for (int u = 0; u < 8; u++) t[u] = win[(msrc + q + u) & CFG::M];
      } else {
#pragma unroll
        for (int u = 0; u < 8; u++) t[u] = __ldcg(dst_al + msrc + q + u);
      }
#pragma unroll
      for (int u = 0; u < 8; u++) win[(mdst + q + u) & CFG::M] = t[u];
    }
  }
  for (; q < ml; q++) {   // tail, or a match that overlaps its own output (offset < 8): byte by byte, in order
    const uint8_t v = near ? win[(msrc + q) & CFG::M] : __ldcg(dst_al + msrc + q);
    win[(mdst + q) & CFG::M] = v;
  }
}

template <class CFG, int PARSE>
__global__ void __launch_bounds__(CFG::WARPS * 32) lz4_decode_kernel(const Lz4Job* jobs, int njobs, unsigned int* error_flag) {
  extern __shared__ __align__(16) uint8_t lz_smem[];
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int job = blockIdx.x * CFG::WARPS + wib;
  if (job >= njobs) return;
  constexpr int TABLES = PARSE == 1 ? 3 * LZ_WP * 2 : 0;   // next / 2-step / 4-step jump tables of the window parse
  uint8_t* win = lz_smem + (size_t)wib * (CFG::WIN + CFG::IN + TABLES);
  uint8_t* in = win + CFG::WIN;
  uint16_t* nx = reinterpret_cast<uint16_t*>(in + CFG::IN);
  uint16_t* j1 = nx + LZ_WP;
  uint16_t* j2 = j1 + LZ_WP;
  const Lz4Job j = jobs[job];
  const unsigned FULL = 0xffffffffu;
  if (j.src_len < 0 || j.dst_len < 0 || j.src_len > 0x7fffffff || j.dst_len > 0x7fffff00) {   // column buffers are < 2 GB
    if (lane == 0) atomicExch(error_flag, 1u);
    return;
  }
  // input positions are "shifted" like the output's: src = j.src rounded down to 16 bytes, so that the 16-byte staging
  // loads are aligned wherever the payload lies (payloads copied as one span keep their host alignment)
  const uint32_t sofs = (uint32_t)(reinterpret_cast<uintptr_t>(j.src) & 15);
  const uint8_t* __restrict__ src = j.src - sofs;
  const uint32_t wofs = (uint32_t)(reinterpret_cast<uintptr_t>(j.dst) & 15);
  uint8_t* dst_al = j.dst - wofs;
  const uint32_t n_src = (uint32_t)j.src_len + sofs, end = (uint32_t)j.dst_len + wofs;
  uint32_t s = sofs, o = wofs, flushed = wofs;
  uint32_t in_hi = 0;   // the input ring holds src[.., in_hi) (multiple of 16), byte p in slot p & CFG::IM
  const bool src_aligned = true;
  bool bad = false, finished = false;

  while (!finished && !bad) {
    // ---- phase A: parse up to 32 short sequences; lane i keeps sequence i ----------------------------------
    uint32_t my_lit_src = 0, my_lit = 0, my_mdst = 0, my_off = 0, my_ml = 0;
    bool my_staged = false;   // this lane's literals are in the input ring
    uint32_t b_lit_src = 0, b_lit = 0, b_off = 0, b_ml = 0;
    bool big = false, b_last = false;
    int n = 0;
    // a whole group of short sequences fits in what is left of the input and the output: stage the input and
    // parse without bounds checks
    const bool safe = src_aligned && n_src - s >= LZ_GROUP_IN && end - o >= LZ_GROUP_OUT;
    if (safe) {
      if (in_hi < (s & ~15u)) in_hi = s & ~15u;
      while (in_hi < s + LZ_GROUP_IN) {   // (the payload allocation is padded: a 16-byte load may run past n_src)
        const uint32_t pos = in_hi + 16u * lane;
        if (pos < n_src) *reinterpret_cast<uint4*>(in + (pos & CFG::IM)) = __ldg(reinterpret_cast<const uint4*>(src + pos));
        in_hi += 512;
      }
      __syncwarp();
    }
    if (PARSE == 1 && safe) {
      // speculative parse of every window position (lane-interleaved: conflict-free byte loads and table stores)
#pragma unroll
      for (int t = 0; t < LZ_WP / 32; t++) {
        const uint32_t p = lane + 32u * t;
        uint32_t a0, a1, a2, a3;
        nx[p] = (uint16_t)lz_spec<CFG>(in, s, p, a0, a1, a2, a3);
      }
      __syncwarp();
#pragma unroll
      for (int t = 0; t < LZ_WP / 32; t++) {   // member after the next one (in-window members only)
        const uint32_t p = lane + 32u * t;
        const uint32_t v = nx[p];
        const uint32_t w = v < (uint32_t)LZ_WP ? nx[v] : LZ_STOP;
        j1[p] = (uint16_t)(w < (uint32_t)LZ_WP ? w : LZ_STOP);
      }
      __syncwarp();
#pragma unroll
      for (int t = 0; t < LZ_WP / 32; t++) {   // four members ahead
        const uint32_t p = lane + 32u * t;
        const uint32_t v = j1[p];
        const uint32_t w = v < (uint32_t)LZ_WP ? j1[v] : LZ_STOP;
        j2[p] = (uint16_t)(w < (uint32_t)LZ_WP ? w : LZ_STOP);
      }
      __syncwarp();
      // anchors: members 0, 4, 8, ... (uniform walk, 8 dependent steps); lanes 4i..4i+3 hang off anchor i
      uint32_t a = 0, my_a = LZ_STOP;
#pragma unroll
      for (int i = 0; i < 8; i++) {
        if ((lane >> 2) == i) my_a = a;
        a = a < (uint32_t)LZ_WP ? j2[a] : LZ_STOP;
      }
      uint32_t pos = LZ_STOP;
      if (my_a < (uint32_t)LZ_WP) {
        const int r = lane & 3;
        if (r == 0) pos = my_a;
        else if (r == 1) pos = nx[my_a];
        else {
          const uint32_t v = j1[my_a];
          pos = r == 2 ? v : (v < (uint32_t)LZ_WP ? nx[v] : LZ_STOP);
        }
        if (pos >= (uint32_t)LZ_WP) pos = LZ_STOP;
      }
      uint32_t f_lit_src = 0, f_lit = 0, f_qoff = 0, f_ml = 0, f_next = LZ_STOP;
      if (pos != LZ_STOP) f_next = lz_spec<CFG>(in, s, pos, f_lit_src, f_lit, f_qoff, f_ml);
      const unsigned vm = __ballot_sync(FULL, pos != LZ_STOP && f_next != LZ_STOP);
      const int nw = vm == FULL ? 32 : __ffs(~vm) - 1;   // the valid lanes are a prefix; anything after the first gap is ignored
      if (nw > 0) {
        const bool mine = lane < nw;
        const uint32_t len = mine ? f_lit + f_ml : 0u;
        uint32_t scan = len;   // inclusive prefix sum of the sequences' output lengths
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t t2 = __shfl_up_sync(FULL, scan, d); if (lane >= d) scan += t2; }
        const uint32_t my_o = o + scan - len;
        const uint32_t off = mine ? ((uint32_t)in[(s + f_qoff) & CFG::IM] | ((uint32_t)in[(s + f_qoff + 1) & CFG::IM] << 8)) : 1u;
        if (__any_sync(FULL, mine && (off == 0 || off > my_o - wofs + f_lit))) { bad = true; break; }
        if (mine) { my_lit_src = s + f_lit_src; my_lit = f_lit; my_mdst = my_o + f_lit; my_off = off; my_ml = f_ml; my_staged = true; }
        o += __shfl_sync(FULL, scan, nw - 1);
        s += __shfl_sync(FULL, f_next, nw - 1);
        n = nw;
      }
    }
    while (n < 32 && !(PARSE == 1 && n > 0)) {   // serial parse (with the window parse: only when it found nothing to take)
      if (safe) {
        const uint32_t token = in[s & CFG::IM];
        uint32_t q = s + 1, lit = token >> 4, ml = token & 15;
        bool ok = true;
        if (lit == 15) { const uint32_t e = in[q & CFG::IM]; q++; lit += e; ok = e != 255 && lit <= (uint32_t)LZ_MAX_LIT; }
        const uint32_t lit_src = q;
        q += lit;
        if (ok) {
          const uint32_t off = (uint32_t)in[q & CFG::IM] | ((uint32_t)in[(q + 1) & CFG::IM] << 8);
          q += 2;
          if (ml == 15) { const uint32_t e = in[q & CFG::IM]; q++; ml += e; ok = e != 255; }
          ml += 4;
          ok = ok && ml <= (uint32_t)LZ_MAX_ML;
          if (ok) {
            if (off == 0 || off > o - wofs + lit) { bad = true; break; }
            if (lane == n) { my_lit_src = lit_src; my_lit = lit; my_mdst = o + lit; my_off = off; my_ml = ml; my_staged = true; }
            s = q;
            o += lit + ml;
            n++;
            continue;
          }
        }
      }
      if (s >= n_src) { finished = true; break; }
      const uint32_t token = __ldg(src + s); s++;
      uint32_t lit = token >> 4;
      if (lit == 15) { uint32_t b; do { if (s >= n_src) { bad = true; break; } b = __ldg(src + s); s++; lit += b; } while (b == 255); }
      if (bad || lit > n_src - s || lit > end - o) { bad = true; break; }
      const uint32_t lit_src = s;
      s += lit;
      const bool last = s >= n_src;   // the block ends with a literals-only sequence
      uint32_t off = 0, ml = 0;
      if (!last) {
        if (n_src - s < 2) { bad = true; break; }
        off = (uint32_t)__ldg(src + s) | ((uint32_t)__ldg(src + s + 1) << 8);
        s += 2;
        ml = token & 15;
        if (ml == 15) { uint32_t b; do { if (s >= n_src) { bad = true; break; } b = __ldg(src + s); s++; ml += b; } while (b == 255); }
        ml += 4;
        if (bad || off == 0 || off > o - wofs + lit || ml > end - o - lit) { bad = true; break; }
      }
      if (lit > LZ_MAX_LIT || ml > LZ_MAX_ML) {   // ends the group; copied by the whole warp below
        big = true; b_lit_src = lit_src; b_lit = lit; b_off = off; b_ml = ml; b_last = last;
        break;
      }
      if (lane == n) { my_lit_src = lit_src; my_lit = lit; my_mdst = o + lit; my_off = off; my_ml = ml; my_staged = false; }
      o += lit + ml;
      n++;
      if (last) { finished = true; break; }
    }
    if (bad) break;

    // ---- phase B: the group's copies -----------------------------------------------------------------------
    if (n > 0) {
      const uint32_t group_end = o;
      if (lane < n) {
        const uint32_t p0 = my_mdst - my_lit;
        if (my_staged) { for (uint32_t k = 0; k < my_lit; k++) win[(p0 + k) & CFG::M] = in[(my_lit_src + k) & CFG::IM]; }
        else { for (uint32_t k = 0; k < my_lit; k++) win[(p0 + k) & CFG::M] = __ldg(src + my_lit_src + k); }
      }
      __syncwarp();
      bool pending = lane < n && my_ml > 0;
      const uint32_t msrc = my_mdst - my_off;
      const uint32_t dep_end = msrc + (my_ml < my_off ? my_ml : my_off);   // exclusive end of the bytes the match needs from others
      const bool near = group_end - msrc <= (uint32_t)CFG::WIN;              // its source is still in the ring after this group's writes
      // Which lanes of this group must have copied their match before mine may run?  Match regions are ordered by lane, so
      // the ones my source range [msrc, dep_end) overlaps are a contiguous run of lower lanes: two 5-step binary searches
      // over the lanes' (start, end) with shuffles.  Literals are all in place already.  A match then waits only for the
      // depth of its own dependency chain (typically 1-3 rounds), not for every earlier lane (it used to be a wavefront).
      const uint32_t my_mend = my_mdst + my_ml;
      uint32_t lo_a = 0, hi_a = lane, lo_b = 0, hi_b = lane;
#pragma unroll
      for (int st = 0; st < 5; st++) {
        const uint32_t mid_a = (lo_a + hi_a) >> 1, mid_b = (lo_b + hi_b) >> 1;
        const uint32_t e = __shfl_sync(FULL, my_mend, (int)(mid_a & 31u));
        const uint32_t b2 = __shfl_sync(FULL, my_mdst, (int)(mid_b & 31u));
        if (lo_a < hi_a) { if (e > msrc) hi_a = mid_a; else lo_a = mid_a + 1; }       // first lane whose match ends beyond msrc
        if (lo_b < hi_b) { if (b2 >= dep_end) hi_b = mid_b; else lo_b = mid_b + 1; }   // first lane whose match starts at / after dep_end
      }
      const uint32_t below_b = lo_b >= 32u ? FULL : ((1u << lo_b) - 1u);
      const uint32_t below_a = lo_a >= 32u ? FULL : ((1u << lo_a) - 1u);
      const uint32_t need = below_b & ~below_a;
      for (;;) {
        const unsigned mask = __ballot_sync(FULL, pending);
        if (!mask) break;
        if (pending && (need & mask) == 0u) {   // the lowest pending lane always qualifies: its needs are lower lanes
          lz_lane_match<CFG>(win, dst_al, my_mdst, msrc, my_ml, my_off, near);
          pending = false;
        }
        __syncwarp();
      }
      lz_flush<CFG>(win, dst_al, flushed, o, lane);
    }
    if (big) {
      // literals, piece by piece: input -> ring -> HBM
      for (uint32_t done = 0; done < b_lit;) {
        const uint32_t piece = b_lit - done < (uint32_t)CFG::PIECE ? b_lit - done : (uint32_t)CFG::PIECE;
        for (uint32_t i = lane; i < piece; i += 32) win[(o + i) & CFG::M] = __ldg(src + b_lit_src + done + i);
        o += piece; done += piece;
        __syncwarp();
        lz_flush<CFG>(win, dst_al, flushed, o, lane);
      }
      // match: byte i comes from [m0 - off, m0): i-th byte of the source for a plain match, the repeating pattern
      // for one that overlaps its own output; bytes that left the ring were flushed and are read back from HBM
      const uint32_t m0 = o;
      for (uint32_t done = 0; done < b_ml;) {
        const uint32_t piece = b_ml - done < (uint32_t)CFG::PIECE ? b_ml - done : (uint32_t)CFG::PIECE;
        const uint32_t piece_end = o + piece;
        if (b_off >= b_ml) {
          for (uint32_t i = lane; i < piece; i += 32) {
            const uint32_t p = m0 - b_off + done + i;
            win[(o + i) & CFG::M] = piece_end - p <= (uint32_t)CFG::WIN ? win[p & CFG::M] : __ldcg(dst_al + p);
          }
        } else {
          for (uint32_t i = lane; i < piece; i += 32) {
            const uint32_t p = m0 - b_off + (done + i) % b_off;
            win[(o + i) & CFG::M] = piece_end - p <= (uint32_t)CFG::WIN ? win[p & CFG::M] : __ldcg(dst_al + p);
          }
        }
        o += piece; done += piece;
        __syncwarp();
        lz_flush<CFG>(win, dst_al, flushed, o, lane);
      }
      if (b_last) finished = true;
    }
  }
  // tail: the last (< 16) bytes of the ring, or everything for a tiny buffer
  __syncwarp();
  if (!bad && o == end) {
    lz_flush<CFG>(win, dst_al, flushed, o, lane);
    for (uint32_t P = flushed + lane; P < end; P += 32) dst_al[P] = win[P & CFG::M];
  } else if (lane == 0) atomicExch(error_flag, 1u);
}

template <class CFG, int PARSE>
static int lz4_launch_cfg(cudaStream_t stream, const Lz4Job* d_jobs, int njobs, unsigned int* d_error) {
  const int blocks = (njobs + CFG::WARPS - 1) / CFG::WARPS;
  constexpr size_t SMEM = CFG::SMEM + (PARSE == 1 ? (size_t)3 * LZ_WP * 2 * CFG::WARPS : 0);
  static bool attr_set[64] = {false};
  int dev = 0;
  SD_CUDA(cudaGetDevice(&dev));
  if (dev < 64 && !attr_set[dev]) {
    SD_CUDA(cudaFuncSetAttribute((lz4_decode_kernel<CFG, PARSE>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM));
    // as many resident buffers per SM as the shared memory allows
    SD_CUDA(cudaFuncSetAttribute((lz4_decode_kernel<CFG, PARSE>), cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
    attr_set[dev] = true;
  }
  lz4_decode_kernel<CFG, PARSE><<<blocks, CFG::WARPS * 32, SMEM, stream>>>(d_jobs, njobs, d_error);
  SD_CUDA(cudaGetLastError());
  return 0;
}

int lz4_launch_shape(cudaStream_t stream, const Lz4Job* d_jobs, int njobs, unsigned int* d_error, bool dense, bool window_parse) {
  if (njobs <= 0) return 0;
  if (window_parse)
    return dense ? lz4_launch_cfg<LzDense, 1>(stream, d_jobs, njobs, d_error) : lz4_launch_cfg<LzDefault, 1>(stream, d_jobs, njobs, d_error);
  return dense ? lz4_launch_cfg<LzDense, 0>(stream, d_jobs, njobs, d_error) : lz4_launch_cfg<LzDefault, 0>(stream, d_jobs, njobs, d_error);
}

int lz4_launch(cudaStream_t stream, const Lz4Job* d_jobs, int njobs, unsigned int* d_error) {
  // defaults: the dense shape (1 warp + ~11 KB of shared memory per CTA: ~19 buffers resident per SM) with the window
  // parse, which expand far more bytes per second with the GPU full of buffers than LzDefault with the serial parse
  static const bool dense = getenv("SD_TUNE_LZ4_DENSE") == nullptr || atoi(getenv("SD_TUNE_LZ4_DENSE")) > 0;
  static const bool wparse = getenv("SD_TUNE_LZ4_PARSE") == nullptr || atoi(getenv("SD_TUNE_LZ4_PARSE")) > 0;
  return lz4_launch_shape(stream, d_jobs, njobs, d_error, dense, wparse);
}

}  // namespace sd

// bench/test hook: the device kernel on raw blocks (include/snappy_gpu.h)
extern "C" int sdx_lz4_expand(int32_t device, const void* const* blocks, const int64_t* block_lens, const int64_t* out_lens,
                              int32_t n, int32_t dst_misalign, int32_t dense, int32_t reps, void* const* outs, double* ms_per_launch) {
  using namespace sd;
  if (n <= 0 || !blocks || !block_lens || !out_lens || dst_misalign < 0 || dst_misalign > 15) return set_error(SD_ERR_INVALID, "sdx_lz4_expand: bad arguments");
  SD_CUDA(cudaSetDevice(device));
  size_t in_total = 0, out_total = 0;
  for (int i = 0; i < n; i++) {
    if (block_lens[i] < 0 || out_lens[i] < 0) return set_error(SD_ERR_INVALID, "sdx_lz4_expand: negative length");
    in_total += ((size_t)block_lens[i] + 16 + 15) & ~size_t(15);
    out_total += ((size_t)out_lens[i] + 32 + 15) & ~size_t(15);
  }
  uint8_t *d_in = nullptr, *d_out = nullptr;
  Lz4Job* d_jobs = nullptr;
  unsigned int* d_err = nullptr;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  int rc = 0;
  std::vector<Lz4Job> jobs((size_t)n);
  auto cleanup = [&]() {
    if (d_in) cudaFree(d_in);
    if (d_out) cudaFree(d_out);
    if (d_jobs) cudaFree(d_jobs);
    if (d_err) cudaFree(d_err);
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
  };
#define LZX(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { rc = set_error(SD_ERR_CUDA, "%s: %s", #call, cudaGetErrorString(e_)); cleanup(); return rc; } } while (0)
  LZX(cudaMalloc(&d_in, in_total + 256));
  LZX(cudaMalloc(&d_out, out_total + 256));
  LZX(cudaMalloc(&d_jobs, sizeof(Lz4Job) * (size_t)n));
  LZX(cudaMalloc(&d_err, 64));
  LZX(cudaMemset(d_err, 0, 64));
  LZX(cudaMemset(d_out, 0xEE, out_total + 256));
  size_t io = 0, oo = 0;
  for (int i = 0; i < n; i++) {
    LZX(cudaMemcpy(d_in + io, blocks[i], (size_t)block_lens[i], cudaMemcpyHostToDevice));
    jobs[i] = Lz4Job{d_in + io, d_out + oo + dst_misalign, block_lens[i], out_lens[i]};
    io += ((size_t)block_lens[i] + 16 + 15) & ~size_t(15);
    oo += ((size_t)out_lens[i] + 32 + 15) & ~size_t(15);
  }
  LZX(cudaMemcpy(d_jobs, jobs.data(), sizeof(Lz4Job) * (size_t)n, cudaMemcpyHostToDevice));
  LZX(cudaEventCreate(&e0));
  LZX(cudaEventCreate(&e1));
  rc = lz4_launch_shape(nullptr, d_jobs, n, d_err, (dense & 1) != 0, (dense & 2) != 0);   // warm-up (and the functional run)
  if (rc) { cleanup(); return rc; }
  LZX(cudaDeviceSynchronize());
  if (reps > 0) {
    LZX(cudaEventRecord(e0, nullptr));
    for (int r = 0; r < reps; r++) { rc = lz4_launch_shape(nullptr, d_jobs, n, d_err, (dense & 1) != 0, (dense & 2) != 0); if (rc) { cleanup(); return rc; } }
    LZX(cudaEventRecord(e1, nullptr));
    LZX(cudaEventSynchronize(e1));
    float ms = 0;
    LZX(cudaEventElapsedTime(&ms, e0, e1));
    if (ms_per_launch) *ms_per_launch = (double)ms / reps;
  }
  unsigned int err = 0;
  LZX(cudaMemcpy(&err, d_err, 4, cudaMemcpyDeviceToHost));
  if (outs) for (int i = 0; i < n; i++) if (outs[i]) LZX(cudaMemcpy(outs[i], jobs[i].dst, (size_t)out_lens[i], cudaMemcpyDeviceToHost));
#undef LZX
  cleanup();
  if (err) return set_error(SD_ERR_INVALID, "sdx_lz4_expand: the device decoder rejected a block");
  return 0;
}

// test hook: host decompression of a stored envelope (LZ4 or Snappy), as used for deltas, delete masks, Snappy columns
extern "C" int sdx_decompress_envelope(const void* buf, int64_t len, void* out, int64_t cap, int64_t* out_len) {
  std::vector<uint8_t> v;
  int rc = sd::decompress_envelope_host(reinterpret_cast<const uint8_t*>(buf), len, v);
  if (rc) return rc;
  if (out_len) *out_len = (int64_t)v.size();
  if ((int64_t)v.size() > cap) return sd::set_error(SD_ERR_OVERFLOW, "output needs %zu bytes", v.size());
  if (!v.empty()) memcpy(out, v.data(), v.size());
  return 0;
}

// test hook: the host prefix decoder (tests/test_lz4_prefix.py compares it with liblz4)
extern "C" int64_t sdx_lz4_decode_prefix(const void* src, int64_t src_len, void* dst, int64_t want) {
  return sd::lz4_decode_prefix(reinterpret_cast<const uint8_t*>(src), src_len, reinterpret_cast<uint8_t*>(dst), want);
}
