// Host replay of kk_convert_f16_kernel launches (KK_LOAD_F16 models).  TEST INFRASTRUCTURE ONLY.
//
// The bf16 replay (kk_dequant_emul.cpp) is included as it is, with every primitive it binds; this file adds what the fp16 instantiation
// of the consumer bodies needs on top of it and plays launches through kk_consume_tile<true>:
//   * pack_f16x2 — fp32 -> fp16 as cvt.rn.f16x2.f32 does it: round to nearest even, overflow to +-inf, fp16 subnormals kept, NaN -> 0x7FFF.
//     The F16C instruction (_cvtss_sh) rounds and the compiler's _Float16 conversion checks it: the two disagreeing fails the run (20).
//     It is declared before the bf16 replay is included, so that the consumer bodies' templates see it where they are defined;
//   * kk_emul_launch_f16 — kk_emul_launch's launch walk with the fp16 consumer dispatch;
//   * the FP8 NaN of the hardware.  The bf16 replay binds kk_f8x2_to_f16x2 to the IEEE widening, which keeps a NaN's sign and payload;
//     an H100's cvt.rn.f16x2.e4m3x2 / .e5m2x2 give 0x7FFF for every NaN of both types instead (all 256 patterns of each, checked by
//     tests/test_gpu_f16.py).  The bf16 path re-packs those halves and cannot tell; the fp16 path stores them as they are.  So after an
//     FP8 tile this replay turns the NaN halves of the tile's own output range into 0x7FFF — every output of such a tile is one
//     conversion result, nothing else is computed from it, and a NaN where the oracle has a number still fails the comparison.
// The product never links this file and has no CPU path.
#include <immintrin.h>

#include <cstdint>

namespace {
inline uint32_t pack_f16x2(float a, float b);
}

#include "kk_dequant_emul.cpp"

namespace {

inline uint32_t f16_rne(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7FFFFFFFu) > 0x7F800000u) return 0x7FFFu;
  const uint32_t h = _cvtss_sh(f, _MM_FROUND_TO_NEAREST_INT) & 0xFFFFu;
  const _Float16 x = (_Float16)f;
  uint16_t hb;
  memcpy(&hb, &x, 2);
  if (hb != (uint16_t)h) flag(20);
  return h;
}
inline uint32_t pack_f16x2(float a, float b) { return f16_rne(a) | (f16_rne(b) << 16); }

// play_tile of kk_dequant_emul.cpp, with the fp16 instantiation of the consumer dispatch
void play_tile_f16(const Dsts& D, const KKTileDesc& t, const Launch& L, uint32_t it) {
  for (g.pass = 1; g.pass <= 2; ++g.pass)
    for (int ctid = 0; ctid < kConsumerThreads; ++ctid) {
      g.warp = ctid >> 5;
      g.lane = ctid & 31;
      g.shfl_calls = 0;
      kk_consume_tile<true>(D, t, 0, t.pay_off, L, g.warp, g.lane, ctid, it);
    }
  g.pass = 0;
}

// The hardware's FP8 NaN (see the top of the file) over the output halves of FP8 tile t in every destination pool.
void canonical_f8_nan(const KKTileDesc& t, uint8_t* const* dst, uint32_t n_dst) {
  if (t.op != KK_OP_F8E4M3_BF16 && t.op != KK_OP_F8E5M2_BF16) return;
  for (uint32_t d = 0; d < n_dst; ++d)
    for (uint64_t k = 0; k < t.n_units; ++k) {
      uint16_t h;
      memcpy(&h, dst[d] + t.dst_off + 2 * k, 2);
      if ((h & 0x7FFFu) > 0x7C00u) {
        h = 0x7FFFu;
        memcpy(dst[d] + t.dst_off + 2 * k, &h, 2);
      }
    }
}

}  // namespace

// kk_emul_launch (same arguments, same checks and failure codes) playing the fp16 instantiation: what launch_convert runs for a launch
// with KK_LAUNCH_F16.  Without statistics: the fp16 tiles make the same loads and stores as the bf16 ones.
extern "C" int kk_emul_launch_f16(const uint8_t* src, uint64_t src_bytes, const KKSeg* segs, uint32_t n_segs, uint32_t n_tiles, uint32_t flags,
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
  if (stats) memset(stats, 0, 5 * sizeof *stats);
  uint32_t cur = 0;
  for (uint32_t tile = 0; tile < n_tiles; ++tile) {
    cur = kk_tile_seg(tile_begin.data(), n_segs, cur, tile);
    const KKSeg& seg = segs[cur];
    if (tile < seg.tile_begin) return 9;
    KKTileDesc d;
    KKTileLoad ld;
    kk_make_tile(seg, tile - seg.tile_begin, kSrcAddr, flags, d, ld);
    memset(stage, 0xEE, sizeof stage);
    g = Emu{};
    uint32_t issued = 0;
    kk_load_tile(ld, Stage{stage, src, src_bytes, ld.tx - d.pay_off - ld.pay, &issued});
    if (g.err) return g.err;
    if (issued != ld.tx) return 12;
    g.tile = stage; g.wtile = stage; g.tile_bytes = ld.kind ? d.pay_off + ld.pay : kStageBytes;
    g.out = dst[0]; g.out_bytes = pool_bytes; g.hits = hits; g.out_mask = mask2; g.byte_mask = mask1;
    g.n_more = (int)n_dst - 1;
    for (int i = 0; i < g.n_more; ++i) g.more_out[i] = dst[i + 1];
    g.src_end = src + src_bytes;
    if (d.op == KK_OP_ROWSPLIT && (!d.C || !d.R)) return 18;
    if (d.bulk == 1 || d.bulk == 3) {
      kk_store_tile(D, d, d.pay_off, L);
      if (g.err) return g.err;
      if (d.bulk == 3 && rs_tiles) ++rs_tiles[0];
      continue;
    }
    play_tile_f16(D, d, L, tile);
    if (g.err) return g.err;
    canonical_f8_nan(d, dst, n_dst);
    if (d.op == KK_OP_ROWSPLIT && rs_tiles) ++rs_tiles[1];
  }
  return 0;
}

// The two packs as the replays bind them, for n floats (n even) -> n 16-bit outputs; returns the failure code (20: the host fp16
// conversions disagree).  The tests hold them against numpy.
extern "C" int kk_emul_pack(int f16, const float* in, uint16_t* out, uint64_t n) {
  g = Emu{};
  for (uint64_t i = 0; i + 1 < n; i += 2) {
    const uint32_t r = f16 ? pack_f16x2(in[i], in[i + 1]) : pack_bf16x2(in[i], in[i + 1]);
    out[i] = (uint16_t)(r & 0xFFFFu);
    out[i + 1] = (uint16_t)(r >> 16);
  }
  return g.err;
}
