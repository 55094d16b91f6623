// Host replay of kk_convert_kernel launches.  TEST INFRASTRUCTURE ONLY.
//
// Compiles kukeon_b200/csrc/kk_consume_tile.cuh — the kernel's per-tile walk (the producer's copies, the bulk stores, the consumer
// dispatch) and the consumer bodies it calls, the exact device source — with g++ by binding the handful of primitives they use
// (bulk copies, shared-memory loads, single-rounding fp32 arithmetic, bf16 packing, the stores) to plain C++, then plays whole
// launches through it (kk_emul_launch), all 16 consumer warps x 32 lanes of every tile (play_tile).  What this checks, on the CPU
// test tier, is the part of the kernel that is easy to get wrong and cannot be seen by reading a formula: which tile the producer
// builds and which bytes it stages, which op runs which body with which arguments, which lane reads which bytes of which block
// and where its output bytes land.  The bindings are stricter than the hardware: a misaligned copy, 16/32-bit shared load or
// bulk store, a read outside the tile's staged payload, a store outside the pool or two stores to the same bytes all fail the
// run.  It does not check PTX spelling or memory ordering; the -m gpu parity tests do.  The product never links this file and
// has no CPU path.
#include <cmath>
#include <cstdint>
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../kukeon_b200/csrc/kk_iq_grids.h"
#include "../../kukeon_b200/csrc/kk_tile.h"

namespace {

constexpr int kConsumerWarps = KK_CONSUMER_WARPS;
constexpr int kConsumerThreads = kConsumerWarps * 32;

struct uint4 { uint32_t x, y, z, w; };
struct uint2 { uint32_t x, y; };
inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return uint4{x, y, z, w}; }

struct Emu {
  const uint8_t* tile = nullptr;  // the stage buffer; shared-memory address a <-> tile[a]
  uint8_t* wtile = nullptr;       // same buffer when the code under test may store into it (sts16 / sts32)
  std::vector<uint32_t>* trace = nullptr;  // when set: every 16/32-bit shared load appends its address (bank-conflict accounting)
  std::vector<uint64_t>* strace = nullptr; // when set: every 16-byte store appends its destination offset (store-transaction accounting)
  uint32_t tile_bytes = 0;
  uint8_t* out = nullptr;         // destination pool 0 (the one hits / masks describe)
  uint8_t* more_out[KK_MAX_DST - 1] = {};  // further destination pools of a fan-out launch: every store is replicated into them
  int n_more = 0;
  uint64_t out_bytes = 0;
  uint8_t* hits = nullptr;  // one counter per 16 output bytes
  uint8_t* out_mask = nullptr;  // per 2 output bytes: written by a scalar (tail) store (per byte for store1_all: see byte_mask)
  uint8_t* byte_mask = nullptr; // per output byte: written by store1_all
  const uint8_t* src_end = nullptr;  // when set: kk_ldg8 must read below it (the end of the staged chunk)
  // the pass of play_tile (1 record, 2 replay: see __shfl_sync below) and the thread it is playing
  static constexpr int kMaxShfl = 64;
  int pass = 0, shfl_calls = 0, warp = 0, lane = 0;
  int err = 0;              // first failure: 1 load out of range, 2 misaligned load, 3 store out of range/misaligned, 4 double store
};
thread_local Emu g;
thread_local float shfl_table[kConsumerWarps][Emu::kMaxShfl][32];  // per warp: the k-th shuffle / vote operand of every lane

inline void flag(int e) { if (!g.err) g.err = e; }
inline uint32_t lds8(uint32_t a) {
  if (a >= g.tile_bytes) { flag(1); return 0; }
  return g.tile[a];
}
inline uint32_t lds16(uint32_t a) {
  if (a & 1u) { flag(2); return 0; }
  if (a + 2 > g.tile_bytes) { flag(1); return 0; }
  if (g.trace) g.trace->push_back(a);
  uint16_t v; memcpy(&v, g.tile + a, 2); return v;
}
inline uint32_t lds32(uint32_t a) {
  if (a & 3u) { flag(2); return 0; }
  if (a + 4 > g.tile_bytes) { flag(1); return 0; }
  if (g.trace) g.trace->push_back(a);
  uint32_t v; memcpy(&v, g.tile + a, 4); return v;
}
inline void sts16(uint32_t a, uint32_t v) {
  if ((a & 1u) || a + 2 > g.tile_bytes || !g.wtile) { flag(6); return; }
  uint16_t h = (uint16_t)v; memcpy(g.wtile + a, &h, 2);
}
inline void sts32(uint32_t a, uint32_t v) {
  if ((a & 3u) || a + 4 > g.tile_bytes || !g.wtile) { flag(6); return; }
  memcpy(g.wtile + a, &v, 4);
}
inline uint2 lds64(uint32_t a) {
  uint2 v{0, 0};
  if (a & 7u) { flag(2); return v; }
  if (a + 8 > g.tile_bytes) { flag(1); return v; }
  memcpy(&v, g.tile + a, 8);
  return v;
}
// Warp shuffle by record / replay: play_tile runs every thread of a tile twice.  Pass 1 (g.pass == 1) records the value each lane offers
// at its k-th shuffle and suppresses pool stores; pass 2 hands out the recorded value of the source lane of the same warp.  Valid for code
// whose shuffled values do not depend on earlier shuffle results and whose lanes all execute the same shuffles (true of q4k_quad).
inline float __shfl_sync(unsigned, float v, int src) {
  if (g.shfl_calls >= Emu::kMaxShfl) { flag(7); return v; }
  float* op = shfl_table[g.warp][g.shfl_calls++];
  if (g.pass == 1) op[g.lane] = v;
  return g.pass == 1 ? v : op[src & 31];
}
// Warp vote, by the same record / replay: pass 1 records every lane's predicate (and returns it: both arms of a vote-guarded branch must
// issue the same shuffles, which they do — the vote only selects the arithmetic), pass 2 returns the AND over the 32 lanes.
inline bool kk_all(bool p) {
  if (g.shfl_calls >= Emu::kMaxShfl) { flag(7); return p; }
  float* op = shfl_table[g.warp][g.shfl_calls++];
  if (g.pass == 1) {
    op[g.lane] = p ? 1.0f : 0.0f;
    return p;
  }
  bool all = true;
  for (int l = 0; l < 32; ++l) all = all && op[l] != 0.0f;
  return all;
}
inline uint32_t kk_f2bits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
inline uint32_t kk_popc(uint32_t u) { return (uint32_t)__builtin_popcount(u); }
inline uint32_t kk_funnel_r(uint32_t lo, uint32_t hi, uint32_t sh) {
  sh &= 31u;
  return sh ? (lo >> sh) | (hi << (32u - sh)) : lo;
}
// Aligned word that starts inside the payload and may end up to 3 bytes behind it: on the device those bytes are whatever the stage's
// slack holds, so here they are poison — a result that depends on them fails the comparison with the oracle.
inline uint32_t lds32_slack(uint32_t a) {
  if (a & 3u) { flag(2); return 0; }
  if (a >= g.tile_bytes) { flag(1); return 0; }
  if (g.trace) g.trace->push_back(a);
  uint32_t v = 0;
  for (uint32_t k = 0; k < 4; ++k) v |= (uint32_t)(a + k < g.tile_bytes ? g.tile[a + k] : (uint8_t)(0xA5u ^ (a + k))) << (8 * k);
  return v;
}
const uint64_t kGridIq2xxs[KK_GRID_IQ2XXS_SIZE] = {KK_GRID_IQ2XXS_VALUES};
const uint64_t kGridIq2xs[KK_GRID_IQ2XS_SIZE] = {KK_GRID_IQ2XS_VALUES};
const uint64_t kGridIq2s[KK_GRID_IQ2S_SIZE] = {KK_GRID_IQ2S_VALUES};
const uint32_t kGridIq3xxs[KK_GRID_IQ3XXS_SIZE] = {KK_GRID_IQ3XXS_VALUES};
const uint32_t kGridIq3s[KK_GRID_IQ3S_SIZE] = {KK_GRID_IQ3S_VALUES};
const uint64_t kGridIq1s[KK_GRID_IQ1S_SIZE] = {KK_GRID_IQ1S_VALUES};
// an index outside the table is a bug in the code under test, not something to read through
inline uint64_t kk_grid_iq2xxs(uint32_t i) { if (i >= KK_GRID_IQ2XXS_SIZE) { flag(8); return 0; } return kGridIq2xxs[i]; }
inline uint64_t kk_grid_iq2xs(uint32_t i) { if (i >= KK_GRID_IQ2XS_SIZE) { flag(8); return 0; } return kGridIq2xs[i]; }
inline uint64_t kk_grid_iq2s(uint32_t i) { if (i >= KK_GRID_IQ2S_SIZE) { flag(8); return 0; } return kGridIq2s[i]; }
inline uint32_t kk_grid_iq3xxs(uint32_t i) { if (i >= KK_GRID_IQ3XXS_SIZE) { flag(8); return 0; } return kGridIq3xxs[i]; }
inline uint32_t kk_grid_iq3s(uint32_t i) { if (i >= KK_GRID_IQ3S_SIZE) { flag(8); return 0; } return kGridIq3s[i]; }
inline uint64_t kk_grid_iq1s(uint32_t i) { if (i >= KK_GRID_IQ1S_SIZE) { flag(8); return 0; } return kGridIq1s[i]; }
inline uint32_t kk_ldg8(const uint8_t* p) {
  if (g.src_end && p >= g.src_end) { flag(11); return 0; }
  return *p;
}
// PRMT (default mode) as the code under test uses it: selector nibble k (low 16 bits; the hardware ignores the rest) picks byte
// (nibble & 7) of {b:a}.  Bit 3 of a nibble asks the hardware to replicate the byte's sign bit instead — never what this code wants, so a
// selector that has it set is a failure (9), not something to mask away.
inline uint32_t kk_byte_perm(uint32_t a, uint32_t b, uint32_t sel) {
  if (sel & 0x8888u) flag(9);
  const uint64_t v = ((uint64_t)b << 32) | a;
  uint32_t r = 0;
  for (int k = 0; k < 4; ++k) r |= (uint32_t)((v >> (8 * ((sel >> (4 * k)) & 7u))) & 0xFFu) << (8 * k);
  return r;
}
inline float kk_bits2f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
inline float kk_fma(float a, float b, float c) { return std::fmaf(a, b, c); }  // correctly rounded single rounding (glibc, -ffp-contract=off)
inline float kk_h2f(uint32_t h) {
  uint16_t b = (uint16_t)h;
  _Float16 x; memcpy(&x, &b, 2);
  return (float)x;
}
inline void kk_h2x2f(uint32_t w, float& x, float& y) { x = kk_h2f(w & 0xFFFFu); y = kk_h2f(w >> 16); }
// one IEEE operation each; -ffp-contract=off in the build line, volatile as a second guard
inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }
inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
inline float __fsub_rn(float a, float b) { volatile float r = a - b; return r; }
inline uint32_t bf16_rne(float f) {
  uint32_t u; memcpy(&u, &f, 4);
  if ((u & 0x7FFFFFFFu) > 0x7F800000u) return 0x7FFFu;  // cvt.rn.bf16x2.f32: canonical NaN
  return (u + 0x7FFFu + ((u >> 16) & 1u)) >> 16;
}
inline uint32_t pack_bf16x2(float a, float b) { return bf16_rne(a) | (bf16_rne(b) << 16); }

struct Dsts { uint32_t n; };  // destination pools: g.out, then g.more_out
// hits[u] counts the BYTES stored into 16-byte unit u: 16 after exactly one vector store (or eight 2-byte tail stores)
inline void store16_all(const Dsts&, uint64_t off, const uint4& v) {
  if (g.pass == 1) return;
  if ((off & 15u) || off + 16 > g.out_bytes) { flag(3); return; }
  if (g.hits[off >> 4]) flag(4);
  g.hits[off >> 4] += 16;
  if (g.strace) g.strace->push_back(off);
  memcpy(g.out + off, &v, 16);
  for (int i = 0; i < g.n_more; ++i) memcpy(g.more_out[i] + off, &v, 16);
}
inline void store1_all(const Dsts&, uint64_t off, uint8_t v) {
  if (g.pass == 1) return;
  if (off + 1 > g.out_bytes) { flag(3); return; }
  if (g.byte_mask[off]) flag(4);
  g.byte_mask[off] = 1;
  g.hits[off >> 4] += 1;
  g.out[off] = v;
  for (int i = 0; i < g.n_more; ++i) g.more_out[i][off] = v;
}
inline void store2_all(const Dsts&, uint64_t off, uint16_t v) {
  if (g.pass == 1) return;
  if ((off & 1u) || off + 2 > g.out_bytes) { flag(3); return; }
  if (g.out_mask[off >> 1]) flag(4);
  g.out_mask[off >> 1] = 1;
  g.hits[off >> 4] += 2;
  memcpy(g.out + off, &v, 2);
  for (int i = 0; i < g.n_more; ++i) memcpy(g.more_out[i] + off, &v, 2);
}
inline void store8_all(const Dsts&, uint64_t off, uint32_t lo, uint32_t hi) {  // half an output vector: four entries of the 2-byte mask
  if (g.pass == 1) return;
  if ((off & 7u) || off + 8 > g.out_bytes) { flag(3); return; }
  for (int k = 0; k < 4; ++k) {
    if (g.out_mask[(off >> 1) + k]) flag(4);
    g.out_mask[(off >> 1) + k] = 1;
  }
  g.hits[off >> 4] += 8;
  const uint32_t v[2] = {lo, hi};
  memcpy(g.out + off, v, 8);
  for (int i = 0; i < g.n_more; ++i) memcpy(g.more_out[i] + off, v, 8);
}
inline void store4_all(const Dsts&, uint64_t off, uint32_t v) {  // one 32-bit element (verbatim transposes): two entries of the 2-byte mask
  if (g.pass == 1) return;
  if ((off & 3u) || off + 4 > g.out_bytes) { flag(3); return; }
  if (g.out_mask[off >> 1] || g.out_mask[(off >> 1) + 1]) flag(4);
  g.out_mask[off >> 1] = g.out_mask[(off >> 1) + 1] = 1;
  g.hits[off >> 4] += 4;
  memcpy(g.out + off, &v, 4);
  for (int i = 0; i < g.n_more; ++i) memcpy(g.more_out[i] + off, &v, 4);
}
// Bulk store of `bytes` from the stage to pool d (t.bulk == 1): 16-byte aligned at both ends and in size, inside the pool and the staged
// payload (else 13).  Pool 0's hit counters count it like every other store.
inline void store_bulk(const Dsts&, int d, uint64_t off, uint32_t src, uint32_t bytes) {
  if ((off & 15u) || (src & 15u) || (bytes & 15u) || off + bytes > g.out_bytes || src + bytes > g.tile_bytes) { flag(13); return; }
  if (d == 0)
    for (uint32_t u = 0; u < bytes; u += 16) {
      if (g.hits[(off + u) >> 4]) flag(4);
      g.hits[(off + u) >> 4] += 16;
    }
  memcpy((d ? g.more_out[d - 1] : g.out) + off, g.tile + src, bytes);
}
inline uint4 lds128(uint32_t a) {
  uint4 v{0, 0, 0, 0};
  if (a & 15u) { flag(2); return v; }
  if (a + 16 > g.tile_bytes) { flag(1); return v; }
  memcpy(&v, g.tile + a, 16);
  return v;
}
// FP8 -> fp16 bit patterns (what cvt.rn.f16x2.e4m3x2 / .e5m2x2 produce; exact)
inline uint32_t f8_to_f16_bits(uint32_t b, bool e5m2) {
  b &= 0xFFu;
  if (e5m2) return b << 8;
  const uint32_t s = (b >> 7) << 15, e = (b >> 3) & 15u, m = b & 7u;
  if (e == 15 && m == 7) return s | 0x7FFFu;                  // NaN
  if (e == 0) {                                              // subnormal m * 2^-9 -> normal fp16
    if (!m) return s;
    int sh = m >= 4 ? 0 : m >= 2 ? 1 : 2;                    // leading one at bit 2 - sh
    return s | (uint32_t)((8 - sh) << 10) | (((m << (sh + 1)) & 7u) << 7);
  }
  return s | ((e + 8u) << 10) | (m << 7);                    // bias 7 -> 15
}
template <bool E5M2>
inline uint32_t kk_f8x2_to_f16x2(uint32_t v) { return f8_to_f16_bits(v, E5M2) | (f8_to_f16_bits(v >> 8, E5M2) << 16); }

// The launch as kk_consume_tile sees it: the staged chunk (transposes gather from src) and, for KK_OP_ROWSPLIT, the pool of every rank
// (ConvertLaunch::xdst) with its size, 16-byte hit counters and per-byte store mask.
struct Launch {
  const uint8_t* src = nullptr;
  uint8_t* const* xdst = nullptr;
  uint32_t n_xdst = 0;
  const uint64_t* xpool_bytes = nullptr;
  uint8_t* const* xhits = nullptr;
  uint8_t* const* xmask1 = nullptr;
};
// A row-split store of `len` bytes into rank j's pool at `off`: the rank must have a pool, the bytes must lie inside it, and no byte of it may
// have been stored before by any rank's launch.  Returns 0 or the failure code.
int rowsplit_store(const Launch& L, uint32_t j, uint64_t off, const uint8_t* v, uint32_t len) {
  if (j >= L.n_xdst || !L.xdst[j]) return 17;
  if (off > L.xpool_bytes[j] || len > L.xpool_bytes[j] - off) return 15;
  for (uint32_t i = 0; i < len; ++i) {
    if (L.xmask1[j][off + i]) return 4;
    L.xmask1[j][off + i] = 1;
    L.xhits[j][(off + i) >> 4] += 1;
  }
  memcpy(L.xdst[j] + off, v, len);
  return 0;
}
inline void rowsplit_store1(const Launch& L, uint32_t j, uint64_t off, uint8_t v) {
  if (g.pass == 1) return;
  if (int rc = rowsplit_store(L, j, off, &v, 1)) flag(rc);
}
// Bulk store of one row-split piece (t.bulk == 3): 16-byte aligned at both ends and in size and not empty (else 14), inside the staged
// payload (else 16), then rowsplit_store's checks.
inline void rowsplit_store_bulk(const Launch& L, uint32_t j, uint64_t off, uint32_t src, uint32_t len) {
  if ((off & 15u) || (src & 15u) || (len & 15u) || !len) { flag(14); return; }
  if (src + len > g.tile_bytes) { flag(16); return; }
  if (int rc = rowsplit_store(L, j, off, g.tile + src, len)) flag(rc);
}
// The consumer barrier: play_tile has every thread run its stage stores (pass 1) before any thread's consumer reads count (pass 2).
inline void named_bar_consumers() {}

constexpr uint64_t kSrcAddr = 0x100000;  // the launch's src base: only its alignment matters (256 bytes, like the staging buffers)
constexpr uint32_t kStageBytes = KK_TILE_SRC_BYTES + KK_STAGE_PAD;
// A stage as the producer's copies fill it from the staged chunk src[0, src_bytes).  slack: bytes at the end of the tile's copies that are
// not payload (the 16-byte rounding of a kind-1 superset, tx - pay_off - pay; 0 for row copies).  issued: bytes copied so far.
struct Stage {
  uint8_t* buf;
  const uint8_t* src;
  uint64_t src_bytes;
  uint32_t slack;
  uint32_t* issued;
};
// One bulk copy: 16-byte aligned source, destination and size, inside the stage (else 10); it may read up to 15 bytes past the chunk, which
// the planner leaves as slack (else 11), but only its rounding may lie there, never payload (else 19).  Bytes past the chunk stay poison.
inline void bulk_load(const Stage& S, uint32_t so, uint64_t go, uint32_t bytes) {
  if (((kSrcAddr + go) & 15u) || (so & 15u) || (bytes & 15u) || so + bytes > kStageBytes) { flag(10); return; }
  if (go > S.src_bytes || go + bytes > S.src_bytes + 15) { flag(11); return; }
  if (go + bytes > S.src_bytes + S.slack) { flag(19); return; }
  memcpy(S.buf + so, S.src + go, (size_t)std::min<uint64_t>(bytes, S.src_bytes - go));
  *S.issued += bytes;
}

#define KK_DQ_DEV static inline
#define min(a, b) ((a) < (b) ? (a) : (b))
#include "../../kukeon_b200/csrc/kk_consume_tile.cuh"
#undef min

// One tile through kk_consume_tile, the kernel's dispatch, for all kConsumerWarps x 32 consumer threads, in two passes over all of them.
// Pass 1 records every lane's shuffle and vote operands, per warp, and performs the stores into the stage, so a transpose's gather is
// complete before pass 2 reads it; it suppresses pool stores.  Pass 2 replays the shuffles and votes, rewrites the same stage bytes and
// stores.  it: the tile counter the kernel's warp rotation reads.  traces / straces (when given) receive each thread's pass-2 16/32-bit
// shared loads and 16-byte store offsets.
void play_tile(const Dsts& D, const KKTileDesc& t, const Launch& L, uint32_t it, std::vector<std::vector<uint32_t>>* traces,
               std::vector<std::vector<uint64_t>>* straces) {
  for (g.pass = 1; g.pass <= 2; ++g.pass)
    for (int ctid = 0; ctid < kConsumerThreads; ++ctid) {
      g.warp = ctid >> 5;
      g.lane = ctid & 31;
      g.shfl_calls = 0;
      g.trace = g.pass == 2 && traces ? &(*traces)[(size_t)ctid] : nullptr;
      g.strace = g.pass == 2 && straces ? &(*straces)[(size_t)ctid] : nullptr;
      kk_consume_tile(D, t, 0, t.pay_off, L, g.warp, g.lane, ctid, it);
    }
  g.pass = 0;
  g.trace = nullptr;
  g.strace = nullptr;
}

}  // namespace

// Shared-memory wavefronts of per-lane load traces: the k-th recorded load of every lane of a warp is one warp instruction; it needs as
// many wavefronts as the worst bank has distinct 4-byte words (same word = broadcast).  Adds to wavefronts / ideal.
void count_wavefronts(const std::vector<std::vector<uint32_t>>& traces, uint64_t& wavefronts, uint64_t& ideal) {
  for (size_t w = 0; w + 31 < traces.size(); w += 32) {
    size_t longest = 0;
    for (int l = 0; l < 32; ++l) longest = std::max(longest, traces[w + l].size());
    for (size_t k = 0; k < longest; ++k) {
      std::vector<uint32_t> words[32];
      bool any = false;
      for (int l = 0; l < 32; ++l) {
        const auto& tr = traces[w + l];
        if (k >= tr.size()) continue;
        any = true;
        const uint32_t word = tr[k] >> 2;
        auto& v = words[word & 31u];
        if (std::find(v.begin(), v.end(), word) == v.end()) v.push_back(word);
      }
      if (!any) continue;
      size_t worst = 1;
      for (auto& v : words) worst = std::max(worst, v.size());
      wavefronts += worst;
      ideal += 1;
    }
  }
}

// 16-byte store transactions of per-lane store traces: the k-th recorded store of every lane of a warp is one warp instruction; it touches
// as many 128-byte lines and 32-byte sectors as its lanes' offsets span (what the LSU / L2 see as transactions).  Adds to instr / lines /
// sectors.
void count_stores(const std::vector<std::vector<uint64_t>>& traces, uint64_t& instr, uint64_t& lines, uint64_t& sectors) {
  for (size_t w = 0; w + 31 < traces.size(); w += 32) {
    size_t longest = 0;
    for (int l = 0; l < 32; ++l) longest = std::max(longest, traces[w + l].size());
    for (size_t k = 0; k < longest; ++k) {
      std::vector<uint64_t> ls, ss;
      for (int l = 0; l < 32; ++l) {
        const auto& tr = traces[w + l];
        if (k >= tr.size()) continue;
        const uint64_t ln = tr[k] >> 7, sc = tr[k] >> 5;
        if (std::find(ls.begin(), ls.end(), ln) == ls.end()) ls.push_back(ln);
        if (std::find(ss.begin(), ss.end(), sc) == ss.end()) ss.push_back(sc);
      }
      if (ls.empty()) continue;
      instr += 1;
      lines += ls.size();
      sectors += ss.size();
    }
  }
}

// A whole launch of kk_convert_kernel, tile by tile, through the kernel's own functions: the segment lookup (kk_tile_seg), the tile
// (kk_make_tile), its copies into a stage buffer (kk_load_tile, checked by bulk_load; the bytes issued must equal the bytes announced to the
// mbarrier), then the consumer side — the bulk stores of aligned copy and row-split tiles (kk_store_tile), or every other tile through
// kk_consume_tile (play_tile) with the launch's tile counter.  The consumers may read the payload only: the 16-byte rounding of a superset
// behind it is out of range, or poison for lds32_slack.
// src: the staged chunk of src_bytes (its base is taken as 256-byte aligned like the staging buffers); dst[0..n_dst): destination pools of
// pool_bytes each; hits / masks describe dst[0] and ACCUMULATE across calls (the caller zeroes them once per pool).
// xdst[0..n_xdst): the pool of every rank, for KK_OP_ROWSPLIT tiles (ConvertLaunch::xdst); xpool_bytes, xhits and xmask1 are each pool's
// size, 16-byte hit counters and per-byte store mask, shared with the launches of the other ranks so that a byte stored twice across ranks
// fails.  rs_tiles (may be null) accumulates the row-split tiles played: [0] by bulk stores (bulk == 3), [1] by the byte-granular consumer.
// stats (may be null) receives, summed over the tiles played through play_tile: [0] the shared-memory wavefronts of the consumers' 16/32-bit
// loads (count_wavefronts; meaningful when all lanes of a warp execute the same loads — byte and vector loads are not traced), [1] the ideal
// (one per warp load), [2] warp-level 16-byte store instructions, [3] the 128-byte lines and [4] the 32-byte sectors they touch (count_stores).
// Returns 0, a positive failure code, or -1 for a bad destination count.
extern "C" int kk_emul_launch(const uint8_t* src, uint64_t src_bytes, const KKSeg* segs, uint32_t n_segs, uint32_t n_tiles, uint32_t flags,
                              uint8_t* const* dst, uint32_t n_dst, uint64_t pool_bytes, uint8_t* hits, uint8_t* mask2, uint8_t* mask1,
                              uint8_t* const* xdst, uint32_t n_xdst, const uint64_t* xpool_bytes, uint8_t* const* xhits, uint8_t* const* xmask1,
                              uint64_t* rs_tiles, uint64_t* stats) {
  if (n_dst < 1 || n_dst > KK_MAX_DST) return -1;
  Launch L;
  L.src = src; L.xdst = xdst; L.n_xdst = n_xdst; L.xpool_bytes = xpool_bytes; L.xhits = xhits; L.xmask1 = xmask1;
  const Dsts D{n_dst};
  static thread_local uint8_t stage[kStageBytes];
  std::vector<uint32_t> tile_begin(n_segs);
  for (uint32_t i = 0; i < n_segs; ++i) tile_begin[i] = segs[i].tile_begin;
  std::vector<std::vector<uint32_t>> traces(stats ? kConsumerThreads : 0);
  std::vector<std::vector<uint64_t>> straces(stats ? kConsumerThreads : 0);
  if (stats) memset(stats, 0, 5 * sizeof *stats);
  uint32_t cur = 0;
  for (uint32_t tile = 0; tile < n_tiles; ++tile) {
    cur = kk_tile_seg(tile_begin.data(), n_segs, cur, tile);
    const KKSeg& seg = segs[cur];
    if (tile < seg.tile_begin) return 9;  // tile_begin[] not monotone from 0
    KKTileDesc d;
    KKTileLoad ld;
    kk_make_tile(seg, tile - seg.tile_begin, kSrcAddr, flags, d, ld);
    memset(stage, 0xEE, sizeof stage);
    g = Emu{};
    uint32_t issued = 0;
    kk_load_tile(ld, Stage{stage, src, src_bytes, ld.tx - d.pay_off - ld.pay, &issued});
    if (g.err) return g.err;
    if (issued != ld.tx) return 12;  // the mbarrier would never complete (or complete early)
    g.tile = stage; g.wtile = stage; g.tile_bytes = ld.kind ? d.pay_off + ld.pay : kStageBytes;
    g.out = dst[0]; g.out_bytes = pool_bytes; g.hits = hits; g.out_mask = mask2; g.byte_mask = mask1;
    g.n_more = (int)n_dst - 1;
    for (int i = 0; i < g.n_more; ++i) g.more_out[i] = dst[i + 1];
    g.src_end = src + src_bytes;
    if (d.op == KK_OP_ROWSPLIT && (!d.C || !d.R)) return 18;  // the kernel would divide by zero
    if (d.bulk == 1 || d.bulk == 3) {  // one lane bulk-stores the stage
      kk_store_tile(D, d, d.pay_off, L);
      if (g.err) return g.err;
      if (d.bulk == 3 && rs_tiles) ++rs_tiles[0];
      continue;
    }
    play_tile(D, d, L, tile, stats ? &traces : nullptr, stats ? &straces : nullptr);
    if (g.err) return g.err;
    if (stats) {
      count_wavefronts(traces, stats[0], stats[1]);
      count_stores(straces, stats[2], stats[3], stats[4]);
      for (auto& v : traces) v.clear();
      for (auto& v : straces) v.clear();
    }
    if (d.op == KK_OP_ROWSPLIT && rs_tiles) ++rs_tiles[1];
  }
  return 0;
}

// Geometry the kernel and the planner share (kk_ops.h), exported so the test can cross-check the Python-side tables.
extern "C" void kk_emul_block_geom(uint32_t op, uint32_t* block_bytes, uint32_t* out_bytes, uint32_t* tile_blocks) {
  const KKBlockGeom gm = kk_block_geom(op);
  *block_bytes = gm.block_bytes; *out_bytes = gm.out_bytes; *tile_blocks = gm.tile_blocks;
}
