// Consumer bodies of kk_convert_kernel, part 2 (part 1 — copy, casts, Q4_K — is kk_consume_core.cuh):
//   * block dequantisers of every other GGUF type: Q8_0, Q6_K, Q4_0, Q4_1, Q5_0, Q5_1, Q2_K, Q3_K, Q5_K, IQ4_NL, IQ4_XS, MXFP4;
//   * the FP8 -> bf16 widening (safetensors F8_E4M3 / F8_E5M2, opt-in);
//   * the 2-D transposes (8-row tiles) and their gather fallback.
//
// Each function is written from the point of view of ONE lane and touches nothing but the primitives below, which the
// including translation unit provides:
//     uint32_t lds8(a) / lds16(a) / lds32(a)     loads from the staged tile (shared-memory byte address; 16- and 32-bit
//                                                forms need natural alignment)
//     float    kk_h2f(h16)                       fp16 bit pattern -> float (exact)
//     float    __fmul_rn / __fadd_rn / __fsub_rn one IEEE fp32 operation each — never contracted into an FMA, so results are
//                                                bit-identical to gguf-py's numpy arithmetic (oracle/oracle.py)
//     uint32_t pack_bf16x2(a, b)                 two floats -> bf16x2, RNE, NaN -> 0x7FFF
//     void     store16_all(D, off, uint4)        16 output bytes to every destination pool
//     void     store2_all(D, off, u16)           one bf16 (ragged tails); store4_all(D, off, u32): one 32-bit element (verbatim transposes)
//     uint4    lds128(a)                         16-byte aligned vector load
//     uint32_t kk_f8x2_to_f16x2<E5M2>(u16)       two FP8 -> two fp16 (exact; cvt.rn.f16x2.e4m3x2 / .e5m2x2 on the device)
//     float    kk_bits2f(u32)                    bit cast
//     uint32_t kk_byte_perm(a, b, sel)           PRMT: byte (sel & 7) of the 8 bytes {b:a} in the low byte of the result
//     uint32_t kk_f2bits(f), kk_popc(u)          bit cast, population count
//     uint32_t kk_funnel_r(lo, hi, sh)           bits [sh, sh+32) of hi:lo (SHF.R.W); lds32_slack(a): aligned word that may end in the stage's slack
//     uint64_t kk_grid_iq2xxs/iq2xs/iq2s/iq1s(i), uint32_t kk_grid_iq3xxs/iq3s(i)   codebook entry i (kk_iq_grids.h; __ldg on the device)
//     void     sts16(a, v) / sts32(a, v)         stores into the stage (gather fallback of the 8-row transposes)
//     uint32_t kk_ldg8(p)                        one byte from global memory (same fallback)
//     Dsts, uint4, make_uint4, kConsumerWarps, KK_DQ_DEV (function attributes)
// kk_kernels.cu binds them to PTX; tests/emul/kk_dequant_emul.cpp binds them to plain C++ (with alignment and
// write-once checks) and runs all 16 x 32 lanes in a loop, so the lane -> element index arithmetic of exactly this source
// is checked against the oracle on the CPU test tier.  That harness is test infrastructure: the product has no CPU path.
//
// Lane mapping of the dequantisers, same for every type: a lane produces 8 consecutive weights = one 16-byte bf16 store; a warp
// iteration produces 512 contiguous output bytes (256-weight super-blocks: one block; 32-weight blocks: eight blocks).
#pragma once
#include "kk_consume_core.cuh"  // lds32_bytes, to_bf16
#include "kk_ops.h"

// ---- loads of any alignment (blocks of 18..210 bytes are only 2-byte aligned inside a tile, or not at all) -----------
KK_DQ_DEV uint32_t lds32_h(uint32_t a) {  // a is 2-byte aligned (falls back to bytes otherwise)
  if (a & 1u) return lds32_bytes(a);
  return lds16(a) | (lds16(a + 2) << 16);
}
KK_DQ_DEV uint32_t lds16_any(uint32_t a) { return (a & 1u) ? (lds8(a) | (lds8(a + 1) << 8)) : lds16(a); }
KK_DQ_DEV uint32_t lds32_any(uint32_t a) {
  if ((a & 3u) == 0) return lds32(a);
  return lds32_h(a);
}
// Four payload bytes at any address, branch-free: the two aligned words that cover them, funnel-shifted (the scheme of lds64_funnel below;
// the second word is read only when a is unaligned and may end in the stage's slack).
KK_DQ_DEV uint32_t lds32_funnel(uint32_t a) {
  const uint32_t base = a & ~3u, sh = (a & 3u) * 8u;
  const uint32_t w0 = lds32(base), w1 = sh ? lds32_slack(base + 4u) : 0u;
  return kk_funnel_r(w0, w1, sh);
}
// Which of the two a block type wants is a compile-time matter.  Tile payloads start on 8-byte boundaries in every real file (GGUF aligns
// tensor data to >= 8 bytes, tiles are multiples of 16 bytes), so blocks whose size is a multiple of 4 are ALWAYS word aligned and
// lds32_any is one load.  Every other size takes the funnel: branch-free, so all of a block's loads issue back to back.  (Round 1 kept the
// branchy form for the 256-weight blocks of 4k + 2 bytes — their alignment is warp-uniform, so it costs no divergence and one
// instruction less on average — but each of its four loads sat in its own BSSY / BRA / BSYNC region and exposed its shared-memory latency
// separately, which left Q3_K, TQ1_0 and IQ2_XXS latency-bound.)
template <uint32_t BLOCK_BYTES>
KK_DQ_DEV uint32_t lds32_blk(uint32_t a) { return (BLOCK_BYTES % 4u != 0u) ? lds32_funnel(a) : lds32_any(a); }
// Eight payload bytes at ANY address a -> two words: the three aligned words that cover them, funnel-shifted into place (SHF.R.W).
// There are no alignment cases, so the lanes of a warp whose blocks sit at different alignments — eight 17-, 18-, 22- or 34-byte blocks
// per warp iteration — do not diverge (the first version branched three ways: aligned / 2-byte funnel / byte by byte, and such a warp
// executed all three).  The third word is read only when a is unaligned; its last 1-3 bytes may lie behind the payload, inside the
// stage's slack (KK_STAGE_PAD), and are shifted out.  The first word may start up to 3 bytes before a: the previous block, the block
// header, or the tile's alignment skew — staged bytes in every case.
KK_DQ_DEV void lds64_funnel(uint32_t a, uint32_t& q0, uint32_t& q1) {
  const uint32_t base = a & ~3u, sh = (a & 3u) * 8u;
  const uint32_t w0 = lds32(base), w1 = lds32(base + 4u), w2 = sh ? lds32_slack(base + 8u) : 0u;
  q0 = kk_funnel_r(w0, w1, sh);
  q1 = kk_funnel_r(w1, w2, sh);
}
KK_DQ_DEV float lds_f16(uint32_t a) { return kk_h2f(lds16_any(a)); }
KK_DQ_DEV void store_bf16x8(const Dsts& D, uint64_t off, const float (&y)[8]) {
  store16_all(D, off, make_uint4(pack_bf16x2(y[0], y[1]), pack_bf16x2(y[2], y[3]), pack_bf16x2(y[4], y[5]), pack_bf16x2(y[6], y[7])));
}

// Byte k (0..3) of w minus BIAS as an exact float, without I2F: PRMT builds 0x4B0000bb = 2^23 + b, one FADD takes off 2^23 + BIAS.
// Every dequantiser below first assembles four small UNSIGNED values per 32-bit word (SIMD-in-word), then calls this per element.
template <int BIAS>
KK_DQ_DEV float byte_to_float(uint32_t w, int k) {
  // the constant is PRMT's FIRST source: a register operand, loaded once outside the loop, with the selector as the immediate.  With the
  // operands the other way round ptxas kept 0x4B000000 as the immediate and re-materialised the four selectors in registers inside
  // every loop iteration (12 extra instructions per 8 elements in the lattice dequantisers; tools/sass_budget.py).
  return __fsub_rn(kk_bits2f(kk_byte_perm(0x4B000000u, w, 0x3004u | (uint32_t)k)), 8388608.0f + (float)BIAS);
}
// bits 0..3 of x -> bit 0 of bytes 0..3 (the multiplier's four set bits are 7 apart, so no partial products overlap)
KK_DQ_DEV uint32_t spread4(uint32_t x) { return ((x & 0xFu) * 0x00204081u) & 0x01010101u; }

// Q8_0 block (34 B): d f16 | qs[32] int8 -> 32 bf16, y = q * d in fp32 (gguf/quants.py Q8_0.dequantize_blocks).
// Lane l of a warp handles elements 8*(l&3)..+8 of block (l>>2): 8 blocks and 512 contiguous output bytes per iteration.
KK_DQ_DEV void consume_q8_0(const Dsts& D, uint32_t pay, uint32_t nblk, uint64_t dst_off, int cwarp, int lane) {
#pragma unroll 2
  for (uint32_t b0 = (uint32_t)cwarp * 8u; b0 < nblk; b0 += kConsumerWarps * 8u) {
    const uint32_t b = b0 + (uint32_t)(lane >> 2);
    {  // lanes past the last block recompute it (in bounds) and skip the store: no branch around the loads, so two iterations' loads overlap
      const uint32_t blk = pay + min(b, nblk - 1u) * KK_Q8_0_BLOCK_BYTES;
      const float d = kk_h2f(lds16_any(blk));
      const uint32_t qa = blk + 2u + 8u * (uint32_t)(lane & 3);
      uint32_t q0, q1;
      lds64_funnel(qa, q0, q1);
      q0 ^= 0x80808080u;  // int8 -> value + 128, unsigned
      q1 ^= 0x80808080u;
      float y[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) y[e] = __fmul_rn(byte_to_float<128>(e < 4 ? q0 : q1, e & 3), d);
      if (b < nblk)
        store16_all(D, dst_off + (uint64_t)b * 64u + (uint32_t)(lane & 3) * 16u,
                    make_uint4(pack_bf16x2(y[0], y[1]), pack_bf16x2(y[2], y[3]), pack_bf16x2(y[4], y[5]), pack_bf16x2(y[6], y[7])));
    }
  }
}

// Q6_K super-block (210 B): ql[128] | qh[64] | scales[16] int8 | d f16 -> 256 bf16 (gguf/quants.py:552-572):
// element e = 32*g + i (g = 0..7): low nibble source ql[64*(g/4) + 32*(g%2) + i] >> 4*((g%4)/2), high 2 bits
// qh[32*(g/4) + i] >> 2*(g%4); q = (lo | hi<<4) - 32; y = (d * scales[e/16]) * q, both products rounded to fp32.
// Lane l handles the 8 elements e = 8l..8l+7 (g = l>>2, i = 8*(l&3)..+8): one block, 512 output bytes per warp iteration.
KK_DQ_DEV void consume_q6k(const Dsts& D, uint32_t pay, uint32_t nblk, uint64_t dst_off, int cwarp, int lane) {
  const int g = lane >> 2, i0 = 8 * (lane & 3);
  const uint32_t ql_off = 64u * (uint32_t)(g >> 2) + 32u * (uint32_t)(g & 1) + (uint32_t)i0;
  const uint32_t qh_off = 128u + 32u * (uint32_t)(g >> 2) + (uint32_t)i0;
  const int lsh = 4 * ((g & 3) >> 1), hsh = 2 * (g & 3);
#pragma unroll 2
  for (uint32_t b = (uint32_t)cwarp; b < nblk; b += kConsumerWarps) {
    const uint32_t blk = pay + b * KK_Q6K_BLOCK_BYTES;
    const float d = kk_h2f(lds16_any(blk + 208u));
    const int sc = (int)(signed char)lds8(blk + 192u + (uint32_t)(lane >> 1));
    const float dsc = __fmul_rn(d, (float)sc);
    uint32_t l0, l1, h0, h1;
    lds64_funnel(blk + ql_off, l0, l1);
    lds64_funnel(blk + qh_off, h0, h1);
    // four 6-bit values per word: low nibble | high two bits << 4 (q + 32, unsigned)
    const uint32_t w0 = ((l0 >> lsh) & 0x0F0F0F0Fu) | (((h0 >> hsh) & 0x03030303u) << 4);
    const uint32_t w1 = ((l1 >> lsh) & 0x0F0F0F0Fu) | (((h1 >> hsh) & 0x03030303u) << 4);
    float y[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) y[e] = __fmul_rn(dsc, byte_to_float<32>(e < 4 ? w0 : w1, e & 3));
    store16_all(D, dst_off + (uint64_t)b * 512u + (uint32_t)lane * 16u,
                make_uint4(pack_bf16x2(y[0], y[1]), pack_bf16x2(y[2], y[3]), pack_bf16x2(y[4], y[5]), pack_bf16x2(y[6], y[7])));
  }
}

// ---- §8(f4): the 32-weight legacy blocks ------------------------------------------------------------------------------
// Q4_0 (18 B): d f16 | qs[16]                      y = d * (q4 - 8)            (gguf/quants.py:220-231)
// Q4_1 (20 B): d f16 | m f16 | qs[16]              y = (d * q4) + m            (gguf/quants.py:254-267)
// Q5_0 (22 B): d f16 | qh u32 | qs[16]             y = d * (q5 - 16)           (gguf/quants.py:291-308)
// Q5_1 (24 B): d f16 | m f16 | qh u32 | qs[16]     y = (d * q5) + m            (gguf/quants.py:333-352)
// Element e < 16 is the LOW nibble of qs[e], element e >= 16 the HIGH nibble of qs[e-16]; bit 4 of element e is bit e of qh.
// Lane l handles elements e0 = 8*(l&3) .. e0+7 of block (l>>2): they come from qs[e0 % 16 .. +8] (one nibble each) and
// the byte (qh >> e0) & 0xFF.  Eight blocks and 512 contiguous output bytes per warp iteration.
template <uint32_t BYTES, bool HAS_M, bool HAS_QH>
KK_DQ_DEV void consume_legacy32(const Dsts& D, uint32_t pay, uint32_t nblk, uint64_t dst_off, int cwarp, int lane) {
  constexpr uint32_t kQhOff = HAS_M ? 4u : 2u;
  constexpr uint32_t kQsOff = kQhOff + (HAS_QH ? 4u : 0u);
  static_assert(kQsOff + 16u == BYTES, "legacy block layout");
  const uint32_t e0 = 8u * (uint32_t)(lane & 3);
  const uint32_t q_off = kQsOff + (e0 & 15u);
  const uint32_t nsh = (e0 >> 4) * 4u;  // 0: low nibbles (elements 0..15), 4: high nibbles (elements 16..31)
#pragma unroll 2
  for (uint32_t b0 = (uint32_t)cwarp * 8u; b0 < nblk; b0 += kConsumerWarps * 8u) {
    const uint32_t b = b0 + (uint32_t)(lane >> 2);
    {  // lanes past the last block recompute it (in bounds) and skip the store: no branch around the loads, so two iterations' loads overlap
      const uint32_t blk = pay + min(b, nblk - 1u) * BYTES;
      const float d = lds_f16(blk);
      const float m = HAS_M ? lds_f16(blk + 2u) : 0.f;
      uint32_t q0, q1;
      lds64_funnel(blk + q_off, q0, q1);
      q0 = (q0 >> nsh) & 0x0F0F0F0Fu;
      q1 = (q1 >> nsh) & 0x0F0F0F0Fu;
      if (HAS_QH) {  // bit 4 of element e0 + k is bit k of this byte of qh
        const uint32_t hbits = (lds32_blk<BYTES>(blk + kQhOff) >> e0) & 0xFFu;
        q0 |= spread4(hbits) << 4;
        q1 |= spread4(hbits >> 4) << 4;
      }
      float y[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        if (HAS_M) y[e] = __fadd_rn(__fmul_rn(d, byte_to_float<0>(e < 4 ? q0 : q1, e & 3)), m);
        else y[e] = __fmul_rn(d, byte_to_float<(HAS_QH ? 16 : 8)>(e < 4 ? q0 : q1, e & 3));
      }
      if (b < nblk) store_bf16x8(D, dst_off + (uint64_t)b * 64u + (uint32_t)(lane & 3) * 16u, y);
    }
  }
}

// ---- §8(f4): the remaining 256-weight K super-blocks; lane l handles elements 8l..8l+7, one block per warp iteration --
// Q2_K (84 B): scales[16] | qs[64] | d f16 | dmin f16  (gguf/quants.py:404-428).  Element e = 128h + 32s + i (h<2, s<4, i<32):
// q = (qs[32h+i] >> 2s) & 3; 16-weight sub-block j = e/16: y = (d*(scales[j]&15))*q - dmin*(scales[j]>>4).
// Lane l: h = l>>4, s = (l>>2)&3, i = 8*(l&3)..+8, j = l>>1.
KK_DQ_DEV void consume_q2k(const Dsts& D, uint32_t pay, uint32_t nblk, uint64_t dst_off, int cwarp, int lane) {
  const uint32_t q_off = 16u + 32u * (uint32_t)(lane >> 4) + 8u * (uint32_t)(lane & 3);
  const uint32_t sh = 2u * (uint32_t)((lane >> 2) & 3);
  // (no `#pragma unroll 2` here: this loop is not latency-bound, and it ran slower unrolled)
  for (uint32_t b = (uint32_t)cwarp; b < nblk; b += kConsumerWarps) {
    const uint32_t blk = pay + b * KK_Q2K_BLOCK_BYTES;
    const float d = lds_f16(blk + 80u), dmin = lds_f16(blk + 82u);
    const uint32_t sc = lds8(blk + (uint32_t)(lane >> 1));
    const float dl = __fmul_rn(d, (float)(sc & 0xFu));
    const float ml = __fmul_rn(dmin, (float)(sc >> 4));
    const uint32_t q0 = (lds32_blk<KK_Q2K_BLOCK_BYTES>(blk + q_off) >> sh) & 0x03030303u;
    const uint32_t q1 = (lds32_blk<KK_Q2K_BLOCK_BYTES>(blk + q_off + 4u) >> sh) & 0x03030303u;
    float y[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) y[e] = __fsub_rn(__fmul_rn(dl, byte_to_float<0>(e < 4 ? q0 : q1, e & 3)), ml);
    store_bf16x8(D, dst_off + (uint64_t)b * 512u + (uint32_t)lane * 16u, y);
  }
}

// Q3_K (110 B): hmask[32] | qs[64] | scales[12] | d f16  (gguf/quants.py:431-472).  Element e = 32g + i (g<8, i<32):
// low bits (qs[32*(g/4) + i] >> 2*(g%4)) & 3; q = low - 4 when bit g of hmask[i] is CLEAR, else low.  Scale k = e/16 is 6 bits:
// low 4 = scales[k] & 15 (k<8) or scales[k-8] >> 4 (k>=8), high 2 = (scales[8 + k%4] >> 2*(k/4)) & 3, value - 32.
// y = (d*scale_k)*q.  Lane l: g = l>>2, i = 8*(l&3)..+8, k = l>>1.
KK_DQ_DEV void consume_q3k(const Dsts& D, uint32_t pay, uint32_t nblk, uint64_t dst_off, int cwarp, int lane) {
  const uint32_t g = (uint32_t)(lane >> 2), i0 = 8u * (uint32_t)(lane & 3), k = (uint32_t)(lane >> 1);
  const uint32_t q_off = 32u + 32u * (g >> 2) + i0;
  const uint32_t sh = 2u * (g & 3u);
  const uint32_t lo_off = 96u + (k & 7u), lo_sh = (k >> 3) * 4u;
  const uint32_t hi_off = 104u + (k & 3u), hi_sh = 2u * (k >> 2);
#pragma unroll 2
  for (uint32_t b = (uint32_t)cwarp; b < nblk; b += kConsumerWarps) {
    const uint32_t blk = pay + b * KK_Q3K_BLOCK_BYTES;
    const float d = lds_f16(blk + 108u);
    const uint32_t lo4 = (lds8(blk + lo_off) >> lo_sh) & 0xFu;
    const uint32_t hi2 = (lds8(blk + hi_off) >> hi_sh) & 0x3u;
    const float dl = __fmul_rn(d, (float)((int)(lo4 | (hi2 << 4)) - 32));
    // q = low - 4 when the mask bit is clear = (low | maskbit << 2) - 4: four 3-bit values per word, bias 4
    const uint32_t w0 = ((lds32_blk<KK_Q3K_BLOCK_BYTES>(blk + q_off) >> sh) & 0x03030303u) | (((lds32_blk<KK_Q3K_BLOCK_BYTES>(blk + i0) >> g) & 0x01010101u) << 2);
    const uint32_t w1 = ((lds32_blk<KK_Q3K_BLOCK_BYTES>(blk + q_off + 4u) >> sh) & 0x03030303u) | (((lds32_blk<KK_Q3K_BLOCK_BYTES>(blk + i0 + 4u) >> g) & 0x01010101u) << 2);
    float y[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) y[e] = __fmul_rn(dl, byte_to_float<4>(e < 4 ? w0 : w1, e & 3));
    store_bf16x8(D, dst_off + (uint64_t)b * 512u + (uint32_t)lane * 16u, y);
  }
}

// Q5_K (176 B): d f16 | dmin f16 | scales[12] | qh[32] | qs[128]  (gguf/quants.py:525-548).  Sub-block j (32 weights), element i:
// q = ((qs[32*(j/2) + i] >> 4*(j%2)) & 15) | (((qh[i] >> j) & 1) << 4); (scale, min) of sub-block j packed as in Q4_K;
// y = (d*sc_j)*q - dmin*m_j.  Implemented by consume_q5k in kk_consume_core.cuh: Q4_K's four-blocks-per-iteration quads with a fifth bit.

// ---- §8(f4): FP8 (safetensors F8_E4M3 / F8_E5M2) widened to bf16, opt-in through KK_LOAD_F8_TO_BF16 -----------------------------
// Elementwise and exact: FP8 -> fp16 with the hardware pair conversion, fp16 -> fp32 -> bf16 (RNE never rounds: every FP8 value
// has at most 3 mantissa bits).  A thread turns 16 source bytes into two 16-byte stores; n = elements of the tile.
template <bool E5M2>
KK_DQ_DEV void f8x4_to_bf16x4(uint32_t w, uint32_t& o0, uint32_t& o1) {  // 4 FP8 in a word -> 2 + 2 bf16
  const uint32_t h0 = kk_f8x2_to_f16x2<E5M2>(w & 0xFFFFu), h1 = kk_f8x2_to_f16x2<E5M2>(w >> 16);
  o0 = pack_bf16x2(kk_h2f(h0 & 0xFFFFu), kk_h2f(h0 >> 16));
  o1 = pack_bf16x2(kk_h2f(h1 & 0xFFFFu), kk_h2f(h1 >> 16));
}
template <bool E5M2>
KK_DQ_DEV void consume_f8(const Dsts& D, uint32_t pay, uint32_t n, uint64_t dst_off, int ctid) {
  const uint32_t ngrp = n >> 4;  // 16 elements -> 32 B out
  const bool al = (pay & 15u) == 0;
  for (uint32_t g = (uint32_t)ctid; g < ngrp; g += kConsumerWarps * 32u) {
    uint32_t w[4];
    if (al) {
      const uint4 v = lds128(pay + (g << 4));
      w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k) w[k] = lds32_any(pay + (g << 4) + 4u * (uint32_t)k);
    }
    uint32_t o[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) f8x4_to_bf16x4<E5M2>(w[k], o[2 * k], o[2 * k + 1]);
    store16_all(D, dst_off + ((uint64_t)g << 5), make_uint4(o[0], o[1], o[2], o[3]));
    store16_all(D, dst_off + ((uint64_t)g << 5) + 16u, make_uint4(o[4], o[5], o[6], o[7]));
  }
  const uint32_t tail = n & 15u, base = ngrp << 4;
  if ((uint32_t)ctid < tail) {
    const uint32_t h = kk_f8x2_to_f16x2<E5M2>(lds8(pay + base + (uint32_t)ctid));
    store2_all(D, dst_off + 2ull * (base + (uint32_t)ctid), (uint16_t)(pack_bf16x2(kk_h2f(h & 0xFFFFu), 0.f) & 0xFFFFu));
  }
}

// ---- 2-D transposes on 8-row tiles (KK_OP_T_*) ---------------------------------------------------------------------------------------
// The stage holds nr <= 8 source rows of nc columns, row r at sbase + r * pitch (staged by the producer's bulk copies, or gathered
// by t_gather when the source rows are not 16-byte aligned).  Thread t takes columns t, t + 512, ...: its 8 loads walk DOWN one
// column while the lanes of its warp sit side by side ALONG the row — consecutive shared-memory words, conflict-free whatever
// the pitch — and the 8 converted values are the 8 * OES contiguous destination bytes dst[(col0 + c) * R + row0 .. + 8).
template <int ES, int CONV>  // CONV: 0 verbatim 16-bit, 1 f32 -> bf16, 2 f16 -> bf16
KK_DQ_DEV uint32_t t_pack2(uint32_t a, uint32_t b) {
  if (CONV == 1) return pack_bf16x2(kk_bits2f(a), kk_bits2f(b));
  if (CONV == 2) return pack_bf16x2(kk_h2f(a), kk_h2f(b));
  return (a & 0xFFFFu) | (b << 16);
}
template <int ES, int CONV>  // CONV 3: verbatim 32-bit (ES == 4, 4-byte outputs); otherwise 2-byte outputs
KK_DQ_DEV void consume_t(const Dsts& D, uint32_t sbase, uint32_t pitch, uint32_t nr, uint32_t nc, uint32_t R, uint32_t col0, uint32_t row0,
                         uint64_t dst_off, int ctid) {
  constexpr uint32_t OES = CONV == 3 ? 4u : 2u;
  // whole 16-byte stores need every column's 8-row group to start on a 16-byte boundary of the pool
  const bool vec = nr == KK_T_ROWS && ((R * OES) & 15u) == 0 && ((row0 * OES) & 15u) == 0 && (dst_off & 15u) == 0;
  for (uint32_t c = (uint32_t)ctid; c < nc; c += kConsumerWarps * 32u) {
    uint32_t v[KK_T_ROWS];
#pragma unroll
    for (uint32_t k = 0; k < KK_T_ROWS; ++k) {
      const uint32_t a = sbase + k * pitch + c * (uint32_t)ES;
      v[k] = k < nr ? (ES == 4 ? lds32(a) : lds16(a)) : 0u;
    }
    const uint64_t off = dst_off + ((uint64_t)(col0 + c) * R + row0) * OES;
    if (CONV == 3) {
      if (vec) {
#pragma unroll
        for (uint32_t g = 0; g < KK_T_ROWS / 4u; ++g) store16_all(D, off + 16u * g, make_uint4(v[4 * g], v[4 * g + 1], v[4 * g + 2], v[4 * g + 3]));
      } else {
#pragma unroll
        for (uint32_t k = 0; k < KK_T_ROWS; ++k)
          if (k < nr) store4_all(D, off + 4u * k, v[k]);
      }
    } else if (vec) {
#pragma unroll
      for (uint32_t g = 0; g < KK_T_ROWS / 8u; ++g)
        store16_all(D, off + 16u * g, make_uint4(t_pack2<ES, CONV>(v[8 * g], v[8 * g + 1]), t_pack2<ES, CONV>(v[8 * g + 2], v[8 * g + 3]),
                                                 t_pack2<ES, CONV>(v[8 * g + 4], v[8 * g + 5]), t_pack2<ES, CONV>(v[8 * g + 6], v[8 * g + 7])));
    } else {
#pragma unroll
      for (uint32_t k = 0; k < KK_T_ROWS; ++k)
        if (k < nr) store2_all(D, off + 2u * k, (uint16_t)(t_pack2<ES, CONV>(v[k], 0u) & 0xFFFFu));
    }
  }
}
// Fallback when the producer could not stage the tile with bulk copies (rows not 16-byte aligned / not a whole number of 16-byte
// units): every consumer thread copies elements from global memory into the same [row][col] layout; the caller puts a barrier
// between this and consume_t.  src points at source element (r0, c0); C = source columns of the tensor.
template <int ES>
KK_DQ_DEV void t_gather(const uint8_t* src, uint32_t sbase, uint32_t pitch, uint32_t nr, uint32_t nc, uint32_t C, int ctid) {
  for (uint32_t i = (uint32_t)ctid; i < nr * nc; i += kConsumerWarps * 32u) {
    const uint32_t r = i / nc, c = i - r * nc;
    const uint8_t* p = src + ((uint64_t)r * C + c) * (uint32_t)ES;
    uint32_t w = 0;
#pragma unroll
    for (int k = 0; k < ES; ++k) w |= kk_ldg8(p + k) << (8 * k);
    if (ES == 4) sts32(sbase + r * pitch + c * 4u, w);
    else sts16(sbase + r * pitch + c * 2u, w);
  }
}

// ---- §8(f4): 4-bit codebook types ---------------------------------------------------------------------------------------------------
// IQ4_NL (18 B): d f16 | qs[16] — Q4_0's nibble layout, value = kIQ4NL[q4]                       (gguf/quants.py:1330-1348)
// IQ4_XS (136 B): d f16 | scales_h u16 | scales_l[4] | qs[128]; sub-block j (32 weights): 6-bit scale
//                 ls = ((scales_l[j/2] >> 4(j%2)) & 15) | (((scales_h >> 2j) & 3) << 4), y = (d*(ls-32)) * kIQ4NL[q4]; its elements
//                 i < 16 are the low nibbles of qs[16j + i], i >= 16 the high nibbles of qs[16j + i - 16]   (gguf/quants.py:1351-1380)
// MXFP4 (17 B):   e u8 (E8M0) | qs[16]; y = 2^(e-128) * kMXFP4[q4] (the table holds DOUBLED e2m1 values)   (gguf/quants.py:656-708)
// The 16-entry tables live in four registers each and are read EIGHT indices at a time with PRMT as the lookup instruction: the lane's
// eight 4-bit indices are squeezed into the nibbles of one word (the PRMT selector format), bits 2:0 of every index select a byte from
// the low half {K0,K1} and from the high half {K2,K3} of the table (two PRMTs per four indices), and a third PRMT takes byte e from the
// one or the other according to bit 3 of index e.  18 instructions per eight lookups; one PRMT + compare + select PER INDEX before.
template <int TABLE>  // 0: IQ4_NL values, 1: MXFP4 (e2m1 x 2)
KK_DQ_DEV void lut16x8(uint32_t x0, uint32_t x1, uint32_t& r0, uint32_t& r1) {
  // x0, x1: four indices each, one per byte (0x0i0j0k0l).  r0, r1: the table entries (+ 128, unsigned bytes) in the same byte order.
  // little-endian packing of {-127,-104,-83,-65, -49,-35,-22,-10, 1,13,25,38, 53,69,89,113} and {0,1,2,3, 4,6,8,12, 0,-1,-2,-3, -4,-6,-8,-12},
  // every entry + 128 so that the bytes are unsigned and byte_to_float<128> (PRMT + FADD) yields the signed value
  constexpr uint32_t K0 = (TABLE ? 0x03020100u : 0xBFAD9881u) ^ 0x80808080u, K1 = (TABLE ? 0x0C080604u : 0xF6EADDCFu) ^ 0x80808080u;
  constexpr uint32_t K2 = (TABLE ? 0xFDFEFF00u : 0x26190D01u) ^ 0x80808080u, K3 = (TABLE ? 0xF4F8FAFCu : 0x71594535u) ^ 0x80808080u;
  const uint32_t t0 = x0 | (x0 >> 4), t1 = x1 | (x1 >> 4);            // byte 0 = k<<4 | l, byte 2 = i<<4 | j
  const uint32_t sel = kk_byte_perm(t0, t1, 0x6420u);                  // nibble e = index e: x0's four in the low half, x1's in the high half
  const uint32_t s7 = sel & 0x77777777u;                               // a selector nibble's bit 3 would ask PRMT for sign replication
  const uint32_t pick = ((sel >> 1) & 0x44444444u) | 0x32103210u;      // nibble e = e + 4 * (bit 3 of index e)
  r0 = kk_byte_perm(kk_byte_perm(K0, K1, s7), kk_byte_perm(K2, K3, s7), pick);  // PRMT reads only the low 16 bits of its selector
  r1 = kk_byte_perm(kk_byte_perm(K0, K1, s7 >> 16), kk_byte_perm(K2, K3, s7 >> 16), pick >> 16);
}
// y[e] = scale * table[index e], one rounding each (gguf-py multiplies the looked-up value by the block scale)
template <int TABLE>
KK_DQ_DEV void codebook8(float scale, uint32_t x0, uint32_t x1, float (&y)[8]) {
  uint32_t r0, r1;
  lut16x8<TABLE>(x0, x1, r0, r1);
#pragma unroll
  for (int e = 0; e < 8; ++e) y[e] = __fmul_rn(scale, byte_to_float<128>(e < 4 ? r0 : r1, e & 3));
}
// 32-weight codebook blocks: lane l takes elements 8(l&3)..+8 of block (l>>2), eight blocks per warp iteration (as consume_legacy32).
template <uint32_t BYTES, int TABLE>
KK_DQ_DEV void consume_codebook32(const Dsts& D, uint32_t pay, uint32_t nblk, uint64_t dst_off, int cwarp, int lane) {
  constexpr uint32_t kQsOff = BYTES - 16u;  // 2 (fp16 d) or 1 (E8M0 byte)
  const uint32_t e0 = 8u * (uint32_t)(lane & 3);
  const uint32_t q_off = kQsOff + (e0 & 15u);
  const uint32_t nsh = (e0 >> 4) * 4u;
#pragma unroll 2
  for (uint32_t b0 = (uint32_t)cwarp * 8u; b0 < nblk; b0 += kConsumerWarps * 8u) {
    const uint32_t b = b0 + (uint32_t)(lane >> 2);
    {  // lanes past the last block recompute it (in bounds) and skip the store: no branch around the loads, so two iterations' loads overlap
      const uint32_t blk = pay + min(b, nblk - 1u) * BYTES;
      float d;
      if (TABLE == 1) {
        const uint32_t e = lds8(blk);
        d = kk_bits2f(e < 2u ? (0x00200000u << e) : ((e - 1u) << 23));  // half of 2^(e-127): the table values are doubled
      } else {
        d = lds_f16(blk);
      }
      uint32_t q0, q1;
      lds64_funnel(blk + q_off, q0, q1);
      q0 = (q0 >> nsh) & 0x0F0F0F0Fu;
      q1 = (q1 >> nsh) & 0x0F0F0F0Fu;
      float y[8];
      codebook8<TABLE>(d, q0, q1, y);
      if (b < nblk) store_bf16x8(D, dst_off + (uint64_t)b * 64u + (uint32_t)(lane & 3) * 16u, y);
    }
  }
}
// IQ4_XS: lane l handles elements 8l..8l+7 = sub-block j = l>>2, i = 8(l&3)..+8; one super-block per warp iteration.
KK_DQ_DEV void consume_iq4xs(const Dsts& D, uint32_t pay, uint32_t nblk, uint64_t dst_off, int cwarp, int lane) {
  const uint32_t j = (uint32_t)(lane >> 2), i0 = 8u * (uint32_t)(lane & 3);
  const uint32_t q_off = 8u + 16u * j + (i0 & 15u);
  const uint32_t nsh = (i0 >> 4) * 4u;
#pragma unroll 2
  for (uint32_t b = (uint32_t)cwarp; b < nblk; b += kConsumerWarps) {
    const uint32_t blk = pay + b * KK_IQ4XS_BLOCK_BYTES;
    const float d = lds_f16(blk);
    const uint32_t sh = lds16_any(blk + 2u);
    const uint32_t sl = lds8(blk + 4u + (j >> 1));
    const uint32_t ls = ((sl >> (4u * (j & 1u))) & 0xFu) | (((sh >> (2u * j)) & 3u) << 4);
    const float dl = __fmul_rn(d, (float)((int)ls - 32));
    const uint32_t q0 = (lds32_blk<KK_IQ4XS_BLOCK_BYTES>(blk + q_off) >> nsh) & 0x0F0F0F0Fu;
    const uint32_t q1 = (lds32_blk<KK_IQ4XS_BLOCK_BYTES>(blk + q_off + 4u) >> nsh) & 0x0F0F0F0Fu;
    float y[8];
    codebook8<0>(dl, q0, q1, y);
    store_bf16x8(D, dst_off + (uint64_t)b * 512u + (uint32_t)lane * 16u, y);
  }
}

// ---- §8(f4): lattice i-quants, ternary types, NVFP4 --------------------------------------------------------------------------------------
// Common shape of the IQ2 / IQ3 types: 8 weights = one codebook entry of 8 unsigned bytes (IQ3: two entries of 4), a sign byte (bit k
// negates weight k) and a group scale db; y = (db * value) * (+-1), which is the product with its sign bit flipped.  Lane l always
// handles weights 8l .. 8l+7 of the super-block (one block per warp iteration), so its 8 outputs are one entry.
KK_DQ_DEV uint32_t ksigns7(uint32_t i7) { return i7 | ((kk_popc(i7) & 1u) << 7); }  // 7 stored bits + their parity (ggml ksigns_iq2xs)
KK_DQ_DEV float signed_mul(float db, uint32_t w, int k, uint32_t signs, int bit) {
  return kk_bits2f(kk_f2bits(__fmul_rn(db, byte_to_float<0>(w, k))) ^ (((signs >> bit) & 1u) << 31));
}
KK_DQ_DEV void store_entry(const Dsts& D, uint64_t off, float db, uint32_t lo, uint32_t hi, uint32_t signs) {
  float y[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) y[e] = signed_mul(db, e < 4 ? lo : hi, e & 3, signs, e);
  store_bf16x8(D, off, y);
}
// db = (d * (0.5 + s)) * K — two roundings, like gguf-py (K is a power of two, the second product is exact)
KK_DQ_DEV float iq_scale(float d, uint32_t s, float k) { return __fmul_rn(__fmul_rn(d, __fadd_rn(0.5f, (float)s)), k); }

// IQ2_XXS (66 B): d f16 | 8 x { u32: four grid indices (bytes) | u32: four 7-bit sign indices, scale in the top 4 bits }
KK_DQ_DEV void consume_iq2xxs(const Dsts& D, uint32_t pay, uint32_t nblk, uint64_t dst_off, int cwarp, int lane) {
  const uint32_t g = (uint32_t)(lane >> 2), k = (uint32_t)(lane & 3);
#pragma unroll 2
  for (uint32_t b = (uint32_t)cwarp; b < nblk; b += kConsumerWarps) {
    const uint32_t blk = pay + b * KK_IQ2XXS_BLOCK_BYTES;
    const float d = lds_f16(blk);
    const uint32_t q1 = lds32_blk<KK_IQ2XXS_BLOCK_BYTES>(blk + 6u + 8u * g);
    const uint64_t grid = kk_grid_iq2xxs(lds8(blk + 2u + 8u * g + k));
    store_entry(D, dst_off + (uint64_t)b * 512u + (uint32_t)lane * 16u, iq_scale(d, q1 >> 28, 0.25f), (uint32_t)grid, (uint32_t)(grid >> 32),
                ksigns7((q1 >> (7u * k)) & 0x7Fu));
  }
}
// IQ2_XS (74 B): d f16 | 32 x u16 { 9-bit grid index | 7-bit sign index } | scales[8] (a nibble per 16 weights)
KK_DQ_DEV void consume_iq2xs(const Dsts& D, uint32_t pay, uint32_t nblk, uint64_t dst_off, int cwarp, int lane) {
  const uint32_t l = (uint32_t)lane;
#pragma unroll 2
  for (uint32_t b = (uint32_t)cwarp; b < nblk; b += kConsumerWarps) {
    const uint32_t blk = pay + b * KK_IQ2XS_BLOCK_BYTES;
    const float d = lds_f16(blk);
    const uint32_t q = lds16_any(blk + 2u + 2u * l);
    const uint32_t s = (lds8(blk + 66u + (l >> 2)) >> (4u * ((l >> 1) & 1u))) & 0xFu;
    const uint64_t grid = kk_grid_iq2xs(q & 511u);
    store_entry(D, dst_off + (uint64_t)b * 512u + l * 16u, iq_scale(d, s, 0.25f), (uint32_t)grid, (uint32_t)(grid >> 32), ksigns7(q >> 9));
  }
}
// IQ2_S (82 B): d f16 | qs[32] | signs[32] | qh[8] (2 more index bits per entry) | scales[8]
KK_DQ_DEV void consume_iq2s(const Dsts& D, uint32_t pay, uint32_t nblk, uint64_t dst_off, int cwarp, int lane) {
  const uint32_t l = (uint32_t)lane;
  // (no `#pragma unroll 2` here: this loop is not latency-bound, and it ran slower unrolled)
  for (uint32_t b = (uint32_t)cwarp; b < nblk; b += kConsumerWarps) {
    const uint32_t blk = pay + b * KK_IQ2S_BLOCK_BYTES;
    const float d = lds_f16(blk);
    const uint32_t idx = lds8(blk + 2u + l) | (((lds8(blk + 66u + (l >> 2)) >> (2u * (l & 3u))) & 3u) << 8);
    const uint32_t s = (lds8(blk + 74u + (l >> 2)) >> (4u * ((l >> 1) & 1u))) & 0xFu;
    const uint64_t grid = kk_grid_iq2s(idx);
    store_entry(D, dst_off + (uint64_t)b * 512u + l * 16u, iq_scale(d, s, 0.25f), (uint32_t)grid, (uint32_t)(grid >> 32), lds8(blk + 34u + l));
  }
}
// IQ3_XXS (98 B): d f16 | qs[64] (one 4-value entry per byte) | 8 x u32 { four 7-bit sign indices, scale in the top 4 bits }
KK_DQ_DEV void consume_iq3xxs(const Dsts& D, uint32_t pay, uint32_t nblk, uint64_t dst_off, int cwarp, int lane) {
  const uint32_t l = (uint32_t)lane, g = l >> 2, k = l & 3u;
#pragma unroll 2
  for (uint32_t b = (uint32_t)cwarp; b < nblk; b += kConsumerWarps) {
    const uint32_t blk = pay + b * KK_IQ3XXS_BLOCK_BYTES;
    const float d = lds_f16(blk);
    const uint32_t w = lds32_blk<KK_IQ3XXS_BLOCK_BYTES>(blk + 66u + 4u * g);
    const uint32_t lo = kk_grid_iq3xxs(lds8(blk + 2u + 2u * l)), hi = kk_grid_iq3xxs(lds8(blk + 3u + 2u * l));
    store_entry(D, dst_off + (uint64_t)b * 512u + l * 16u, iq_scale(d, w >> 28, 0.5f), lo, hi, ksigns7((w >> (7u * k)) & 0x7Fu));
  }
}
// IQ3_S (110 B): d f16 | qs[64] | qh[8] (a ninth index bit per entry) | signs[32] | scales[4] (a nibble per 32 weights); db = d * (1 + 2s)
KK_DQ_DEV void consume_iq3s(const Dsts& D, uint32_t pay, uint32_t nblk, uint64_t dst_off, int cwarp, int lane) {
  const uint32_t l = (uint32_t)lane, g = l >> 2;
#pragma unroll 2
  for (uint32_t b = (uint32_t)cwarp; b < nblk; b += kConsumerWarps) {
    const uint32_t blk = pay + b * KK_IQ3S_BLOCK_BYTES;
    const float d = lds_f16(blk);
    const uint32_t qh = lds8(blk + 66u + (l >> 2));  // entries 2l and 2l+1 live in byte (2l)/8, bits (2l)%8 and +1
    const uint32_t i0 = lds8(blk + 2u + 2u * l) | (((qh >> ((2u * l) & 7u)) & 1u) << 8);
    const uint32_t i1 = lds8(blk + 3u + 2u * l) | (((qh >> (((2u * l) & 7u) + 1u)) & 1u) << 8);
    const uint32_t s = (lds8(blk + 106u + (g >> 1)) >> (4u * (g & 1u))) & 0xFu;
    store_entry(D, dst_off + (uint64_t)b * 512u + l * 16u, __fmul_rn(d, (float)(1u + 2u * s)), kk_grid_iq3s(i0), kk_grid_iq3s(i1), lds8(blk + 74u + l));
  }
}
// IQ1_S / IQ1_M: codebook values in {-1, 0, 1} (stored + 1), y = dl * (value + delta), delta = +-0.125
KK_DQ_DEV void store_entry_iq1(const Dsts& D, uint64_t off, float dl, uint64_t grid, float delta) {
  const uint32_t lo = (uint32_t)grid, hi = (uint32_t)(grid >> 32);
  float y[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) y[e] = __fmul_rn(dl, __fadd_rn(byte_to_float<1>(e < 4 ? lo : hi, e & 3), delta));
  store_bf16x8(D, off, y);
}
// IQ1_S (50 B): d f16 | qs[32] | 8 x u16 { four 3-bit index extensions | 3-bit scale << 12 | delta sign << 15 }
KK_DQ_DEV void consume_iq1s(const Dsts& D, uint32_t pay, uint32_t nblk, uint64_t dst_off, int cwarp, int lane) {
  const uint32_t l = (uint32_t)lane, g = l >> 2, k = l & 3u;
#pragma unroll 2
  for (uint32_t b = (uint32_t)cwarp; b < nblk; b += kConsumerWarps) {
    const uint32_t blk = pay + b * KK_IQ1S_BLOCK_BYTES;
    const float d = lds_f16(blk);
    const uint32_t qh = lds16_any(blk + 34u + 2u * g);
    const uint32_t idx = lds8(blk + 2u + l) | (((qh >> (3u * k)) & 7u) << 8);
    store_entry_iq1(D, dst_off + (uint64_t)b * 512u + l * 16u, __fmul_rn(d, (float)(2u * ((qh >> 12) & 7u) + 1u)), kk_grid_iq1s(idx),
                    (qh & 0x8000u) ? -0.125f : 0.125f);
  }
}
// IQ1_M (56 B): qs[32] | qh[16] (a nibble per entry: 3 index bits, bit 3 = delta sign) | 4 x u16 { four 3-bit scales | a nibble of the fp16 d }
KK_DQ_DEV void consume_iq1m(const Dsts& D, uint32_t pay, uint32_t nblk, uint64_t dst_off, int cwarp, int lane) {
  const uint32_t l = (uint32_t)lane, k16 = l >> 1;
#pragma unroll 2
  for (uint32_t b = (uint32_t)cwarp; b < nblk; b += kConsumerWarps) {
    const uint32_t blk = pay + b * KK_IQ1M_BLOCK_BYTES;
    const uint32_t s0 = lds16_any(blk + 48u), s1 = lds16_any(blk + 50u), s2 = lds16_any(blk + 52u), s3 = lds16_any(blk + 54u);
    const float d = kk_h2f((s0 >> 12) | ((s1 >> 12) << 4) | ((s2 >> 12) << 8) | ((s3 >> 12) << 12));
    const uint32_t sw = (k16 >> 2) == 0 ? s0 : (k16 >> 2) == 1 ? s1 : (k16 >> 2) == 2 ? s2 : s3;
    const uint32_t sc = (sw >> (3u * (k16 & 3u))) & 7u;
    const uint32_t nib = (lds8(blk + 32u + (l >> 1)) >> (4u * (l & 1u))) & 0xFu;
    store_entry_iq1(D, dst_off + (uint64_t)b * 512u + l * 16u, __fmul_rn(d, (float)(2u * sc + 1u)), kk_grid_iq1s(lds8(blk + l) | ((nib & 7u) << 8)),
                    (nib & 8u) ? -0.125f : 0.125f);
  }
}
// TQ2_0 (66 B): qs[64] | d f16; weight 128h + 32s + i = ((qs[32h+i] >> 2s) & 3) - 1 — Q2_K's bit layout without scales
KK_DQ_DEV void consume_tq2_0(const Dsts& D, uint32_t pay, uint32_t nblk, uint64_t dst_off, int cwarp, int lane) {
  const uint32_t q_off = 32u * (uint32_t)(lane >> 4) + 8u * (uint32_t)(lane & 3);
  const uint32_t sh = 2u * (uint32_t)((lane >> 2) & 3);
#pragma unroll 2
  for (uint32_t b = (uint32_t)cwarp; b < nblk; b += kConsumerWarps) {
    const uint32_t blk = pay + b * KK_TQ2_0_BLOCK_BYTES;
    const float d = lds_f16(blk + 64u);
    const uint32_t q0 = (lds32_blk<KK_TQ2_0_BLOCK_BYTES>(blk + q_off) >> sh) & 0x03030303u, q1 = (lds32_blk<KK_TQ2_0_BLOCK_BYTES>(blk + q_off + 4u) >> sh) & 0x03030303u;
    float y[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) y[e] = __fmul_rn(d, byte_to_float<1>(e < 4 ? q0 : q1, e & 3));
    store_bf16x8(D, dst_off + (uint64_t)b * 512u + (uint32_t)lane * 16u, y);
  }
}
// TQ1_0 (54 B): qs[48] | qh[4] | d f16 — base-3 digits: trit = (((B * 3^p) & 255) * 3) >> 8.  Four source bytes are processed as two
// 16-bit lanes per multiply (B * 81 < 2^16): returns the four trits as bytes of one word.
KK_DQ_DEV uint32_t tq1_trits4(uint32_t w, uint32_t m) {
  const uint32_t ev = ((((w & 0x00FF00FFu) * m) & 0x00FF00FFu) * 3u >> 8) & 0x00030003u;         // bytes 0 and 2
  const uint32_t od = (((((w >> 8) & 0x00FF00FFu) * m) & 0x00FF00FFu) * 3u >> 8) & 0x00030003u;  // bytes 1 and 3
  return ev | (od << 8);
}
KK_DQ_DEV void consume_tq1_0(const Dsts& D, uint32_t pay, uint32_t nblk, uint64_t dst_off, int cwarp, int lane) {
  // weights 8l..8l+7: lanes 0-19 read qs[0..31] with power l/4, lanes 20-29 qs[32..47] with power (l-20)/2, lanes 30-31 all of qh with
  // powers 2(l-30) (first four weights) and 2(l-30)+1 (last four)
  const uint32_t l = (uint32_t)lane;
  uint32_t a0, a1, p0, p1;
  if (l < 20u) { a0 = 8u * (l & 3u); a1 = a0 + 4u; p0 = p1 = l >> 2; }
  else if (l < 30u) { a0 = 32u + 8u * ((l - 20u) & 1u); a1 = a0 + 4u; p0 = p1 = (l - 20u) >> 1; }
  else { a0 = a1 = 48u; p0 = 2u * (l - 30u); p1 = p0 + 1u; }
  const uint32_t m0 = (uint32_t)((0x000000511B090301ull >> (8u * p0)) & 0xFFu), m1 = (uint32_t)((0x000000511B090301ull >> (8u * p1)) & 0xFFu);  // 3^p
#pragma unroll 2
  for (uint32_t b = (uint32_t)cwarp; b < nblk; b += kConsumerWarps) {
    const uint32_t blk = pay + b * KK_TQ1_0_BLOCK_BYTES;
    const float d = lds_f16(blk + 52u);
    const uint32_t t0 = tq1_trits4(lds32_blk<KK_TQ1_0_BLOCK_BYTES>(blk + a0), m0), t1 = tq1_trits4(lds32_blk<KK_TQ1_0_BLOCK_BYTES>(blk + a1), m1);
    float y[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) y[e] = __fmul_rn(d, byte_to_float<1>(e < 4 ? t0 : t1, e & 3));
    store_bf16x8(D, dst_off + (uint64_t)b * 512u + l * 16u, y);
  }
}
// NVFP4 (36 B, 64 weights): 4 x UE4M3 scale (one per 16 weights) | qs[32]; sub-block s uses qs[8s..8s+7]: low nibbles = its first 8 weights,
// high nibbles the next 8; y = (scale / 2) * kMXFP4[q4] (doubled e2m1 table).  Lane l: block l>>3 of four per warp iteration, sub-block (l>>1)&3,
// half l&1.
KK_DQ_DEV void consume_nvfp4(const Dsts& D, uint32_t pay, uint32_t nblk, uint64_t dst_off, int cwarp, int lane) {
  const uint32_t l = (uint32_t)lane, sb = (l >> 1) & 3u, nsh = 4u * (l & 1u);
#pragma unroll 2
  for (uint32_t b0 = (uint32_t)cwarp * 4u; b0 < nblk; b0 += kConsumerWarps * 4u) {
    const uint32_t b = b0 + (l >> 3);
    {
      const uint32_t blk = pay + min(b, nblk - 1u) * KK_NVFP4_BLOCK_BYTES;
      const uint32_t x = lds8(blk + sb), e = (x >> 3) & 0xFu, m = x & 7u;
      // half the unsigned-E4M3 value: (1 + m/8) * 2^(e-8) built as bits; e == 0: m * 2^-10; 0x00 and 0x7F decode to 0
      float d = e ? kk_bits2f(((e + 119u) << 23) | (m << 20)) : __fmul_rn((float)m, 0.0009765625f);
      if (x == 0u || x == 0x7Fu) d = 0.0f;
      const uint32_t q0 = (lds32_blk<KK_NVFP4_BLOCK_BYTES>(blk + 4u + 8u * sb) >> nsh) & 0x0F0F0F0Fu, q1 = (lds32_blk<KK_NVFP4_BLOCK_BYTES>(blk + 8u + 8u * sb) >> nsh) & 0x0F0F0F0Fu;
      float y[8];
      codebook8<1>(d, q0, q1, y);
      if (b < nblk) store_bf16x8(D, dst_off + (uint64_t)b * 128u + (l & 7u) * 16u, y);
    }
  }
}
