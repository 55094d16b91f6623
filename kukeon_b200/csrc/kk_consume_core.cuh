// Core consumer bodies of kk_convert_kernel: verbatim copy (register path), fp32 / 16-bit float casts and the Q4_K dequantiser.
// Like kk_dequant.cuh this file is written from the point of view of one lane against primitives the including translation
// unit binds (see the list at the top of kk_dequant.cuh; additionally lds64, store1_all, kk_h2x2f and — for Q4_K, the one
// function here whose lanes trade values — __shfl_sync): PTX in kk_kernels.cu, checked C++ in tests/emul/kk_dequant_emul.cpp,
// where the warp shuffle is emulated by playing every tile twice (record, then replay).
//
// Output format.  Every body that converts is a template on `bool F16`, the launch's 16-bit output format: false packs bf16
// (pack_bf16x2), true IEEE binary16 (pack_f16x2, KK_LAUNCH_F16).  The arithmetic before the pack is the same fp32 in both.
#pragma once
#include "kk_ops.h"

// Two floats -> one packed pair of the output format (a in the low half), round-to-nearest-even, NaN -> 0x7FFF.  The operands' type is a
// template parameter (always float) so that pack_f16x2 is looked up only where the f16 instantiation is made: an includer that plays bf16
// tiles alone need not bind it.
template <bool F16, class F>
KK_DQ_DEV uint32_t pack2(F a, F b) {
  if constexpr (F16) return pack_f16x2(a, b);
  else return pack_bf16x2(a, b);
}
// The 16-bit float that is NOT the output format -> float (exact): the source of KK_OP_F16_BF16 / KK_OP_T_F16_BF16, fp16 in a bf16
// launch and bf16 in an f16 launch.  other16x2_to_f: both halves of a word (low half -> x).
template <bool F16>
KK_DQ_DEV float other16_to_f(uint32_t h) { return F16 ? kk_bits2f(h << 16) : kk_h2f(h); }
template <bool F16>
KK_DQ_DEV void other16x2_to_f(uint32_t w, float& x, float& y) {
  if (F16) {
    x = kk_bits2f(w << 16);
    y = kk_bits2f(w & 0xFFFF0000u);
  } else {
    kk_h2x2f(w, x, y);
  }
}

// ctid: 0..kConsumerThreads-1 within the consumer warps.
KK_DQ_DEV uint32_t lds32_bytes(uint32_t a) { return lds8(a) | (lds8(a + 1) << 8) | (lds8(a + 2) << 16) | (lds8(a + 3) << 24); }
template <bool F16>
KK_DQ_DEV uint16_t to16(float a) { return (uint16_t)(pack2<F16>(a, 0.f) & 0xFFFFu); }


KK_DQ_DEV void consume_copy(const Dsts& D, uint32_t pay, uint32_t n, uint64_t dst_off, int ctid) {
  const uint32_t nvec = n >> 4;
  if ((pay & 15u) == 0) {
    for (uint32_t i = ctid; i < nvec; i += kConsumerThreads) store16_all(D, dst_off + ((uint64_t)i << 4), lds128(pay + (i << 4)));
  } else {
    for (uint32_t i = ctid; i < nvec; i += kConsumerThreads) {
      uint32_t w[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        uint32_t a = pay + (i << 4) + 4 * k;
        w[k] = lds8(a) | (lds8(a + 1) << 8) | (lds8(a + 2) << 16) | (lds8(a + 3) << 24);
      }
      store16_all(D, dst_off + ((uint64_t)i << 4), make_uint4(w[0], w[1], w[2], w[3]));
    }
  }
  const uint32_t tail = n & 15u;
  if (ctid < (int)tail) store1_all(D, dst_off + ((uint64_t)nvec << 4) + ctid, (uint8_t)lds8(pay + (nvec << 4) + ctid));
}

KK_DQ_DEV float lds_f32_any(uint32_t a) {
  uint32_t w;
  if ((a & 3u) == 0) w = lds32(a);
  else w = lds8(a) | (lds8(a + 1) << 8) | (lds8(a + 2) << 16) | (lds8(a + 3) << 24);
  return kk_bits2f(w);
}
template <bool F16>
KK_DQ_DEV float lds_other16_any(uint32_t a) {
  uint32_t h;
  if ((a & 1u) == 0) h = lds16(a);
  else h = lds8(a) | (lds8(a + 1) << 8);
  return other16_to_f<F16>(h);
}

template <bool F16>
KK_DQ_DEV void consume_f32(const Dsts& D, uint32_t pay, uint32_t n, uint64_t dst_off, int ctid) {
  if ((pay & 15u) == 0) {
    // 4 elements per thread and step: one 16-byte load at a 16-byte lane stride (a warp reads 512 contiguous bytes: 4 wavefronts, the minimum)
    // and one 8-byte store (a warp writes 256 contiguous bytes).  Round 1 took 8 elements per thread — two 16-byte loads at a 32-byte lane
    // stride, a 2-way bank conflict on each.
    const uint32_t nq = n >> 2;
    for (uint32_t g = ctid; g < nq; g += kConsumerThreads) {
      const uint4 a = lds128(pay + (g << 4));
      store8_all(D, dst_off + ((uint64_t)g << 3), pack2<F16>(kk_bits2f(a.x), kk_bits2f(a.y)), pack2<F16>(kk_bits2f(a.z), kk_bits2f(a.w)));
    }
    const uint32_t tail = n & 3u, base = nq << 2;
    if (ctid < (int)tail) store2_all(D, dst_off + 2ull * (base + ctid), to16<F16>(lds_f32_any(pay + 4 * (base + ctid))));
    return;
  }
  const uint32_t ngrp = n >> 3;  // 8 elements -> 16 B out
  for (uint32_t g = ctid; g < ngrp; g += kConsumerThreads) {
    float f[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) f[k] = lds_f32_any(pay + (g << 5) + 4 * k);
    store16_all(D, dst_off + ((uint64_t)g << 4),
                make_uint4(pack2<F16>(f[0], f[1]), pack2<F16>(f[2], f[3]), pack2<F16>(f[4], f[5]), pack2<F16>(f[6], f[7])));
  }
  const uint32_t tail = n & 7u, base = ngrp << 3;
  if (ctid < (int)tail) store2_all(D, dst_off + 2ull * (base + ctid), to16<F16>(lds_f32_any(pay + 4 * (base + ctid))));
}

// KK_OP_F16_BF16: the other 16-bit float -> the output format (fp16 -> bf16, or bf16 -> fp16 under KK_LAUNCH_F16)
template <bool F16>
KK_DQ_DEV void consume_f16(const Dsts& D, uint32_t pay, uint32_t n, uint64_t dst_off, int ctid) {
  const uint32_t ngrp = n >> 3;
  if ((pay & 15u) == 0) {
    for (uint32_t g = ctid; g < ngrp; g += kConsumerThreads) {
      uint4 a = lds128(pay + (g << 4));
      const uint32_t w[4] = {a.x, a.y, a.z, a.w};
      uint32_t o[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float fx, fy;
        other16x2_to_f<F16>(w[k], fx, fy);
        o[k] = pack2<F16>(fx, fy);
      }
      store16_all(D, dst_off + ((uint64_t)g << 4), make_uint4(o[0], o[1], o[2], o[3]));
    }
  } else {
    for (uint32_t g = ctid; g < ngrp; g += kConsumerThreads) {
      float f[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) f[k] = lds_other16_any<F16>(pay + (g << 4) + 2 * k);
      store16_all(D, dst_off + ((uint64_t)g << 4),
                  make_uint4(pack2<F16>(f[0], f[1]), pack2<F16>(f[2], f[3]), pack2<F16>(f[4], f[5]), pack2<F16>(f[6], f[7])));
    }
  }
  const uint32_t tail = n & 7u, base = ngrp << 3;
  if (ctid < (int)tail) store2_all(D, dst_off + 2ull * (base + ctid), to16<F16>(lds_other16_any<F16>(pay + 2 * (base + ctid))));
}

// Q4_K super-block (144 B): d f16 | dmin f16 | scales[12] | qs[128]  ->  256 bf16 (fp16 under KK_LAUNCH_F16).
// y = (d*sc_j)*q - (dmin*m_j), every product and the difference rounded to fp32 separately (no FMA
// contraction) so the result is bit-identical to the oracle's gguf-py restatement, then RNE to bf16.
//
// One warp handles FOUR super-blocks per iteration: lane l decodes the 6-bit (scale, min) pair of
// sub-block (l & 7) of block (l >> 3) — so the unpack runs once per four blocks instead of once per block —
// and __shfl_sync hands every lane the pair of the sub-block its 8 outputs belong to.  The four blocks'
// dependency chains are independent and fully unrolled (ILP hides the ALU latency with only 2 warps/SMSP).
// Expansion of one quad.  FAST: c = -(d*sc) * 2^23 (exact: a power-of-two scaling) lets ONE FMA turn the magic-number float 2^23 + q straight
// into the rounded product — fma(dsc, 2^23 + q, c) = round(dsc * q), the same single rounding as __fmul_rn(dsc, (float)q) — instead of
// FADD + FMUL per element (the loop is issue-bound).  The identity
// holds bit for bit only for a finite scale that is not negative: with +-inf the FMA sees inf - inf (NaN, where the two-step form gives
// +-inf for q > 0), and for q = 0 under a negative scale it yields +0 where the product is -0 (visible when the sub-block minimum is 0).
// Real checkpoints have d >= 0 and finite — every quad takes the fast form — but random bytes are part of the parity tests, so the warp
// votes once per quad and a quad with any other scale takes the two-step form.
// Q5: the same quad for Q5_K (176 B: d | dmin | scales[12] | qh[32] | qs[128]) — identical header and scale packing, the nibbles start 32 bytes
// later and element i of sub-block j takes its fifth bit from bit j of qh[i].
template <bool F16, bool ALIGNED, bool FAST, bool Q5>
KK_DQ_DEV void q4k_expand(const Dsts& D, uint32_t pay, uint32_t b0, uint32_t nb, uint64_t dst_off, int lane, float dsc_j, float dsc_c, float dmn_j) {
  constexpr uint32_t BB = Q5 ? 176u : KK_Q4K_BLOCK_BYTES;
  // this lane's 8 outputs of every block live in sub-block myj = lane >> 2
  const int myj = lane >> 2;
  const uint32_t qoff = (Q5 ? 48u : 16u) + 32u * (uint32_t)(myj >> 1) + 8u * (uint32_t)(lane & 3);
  const uint32_t hoff = 16u + 8u * (uint32_t)(lane & 3);
  const int nsh = (myj & 1) * 4;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float dsc = __shfl_sync(0xffffffffu, dsc_j, 8 * k + myj);
    const float dsc2 = __shfl_sync(0xffffffffu, dsc_c, 8 * k + myj);
    const float dmn = __shfl_sync(0xffffffffu, dmn_j, 8 * k + myj);
    if ((uint32_t)k < nb) {
      const uint32_t blk = pay + (b0 + k) * BB;
      const uint32_t qa = blk + qoff;
      uint32_t q0, q1;
      if (ALIGNED) {
        const uint2 q = lds64(qa);
        q0 = q.x; q1 = q.y;
      } else {
        q0 = lds32_bytes(qa); q1 = lds32_bytes(qa + 4);
      }
      q0 = (q0 >> nsh) & 0x0F0F0F0Fu;
      q1 = (q1 >> nsh) & 0x0F0F0F0Fu;
      if (Q5) {
        uint32_t h0, h1;
        if (ALIGNED) {
          const uint2 h = lds64(blk + hoff);
          h0 = h.x; h1 = h.y;
        } else {
          h0 = lds32_bytes(blk + hoff); h1 = lds32_bytes(blk + hoff + 4);
        }
        q0 |= ((h0 >> myj) & 0x01010101u) << 4;
        q1 |= ((h1 >> myj) & 0x01010101u) << 4;
      }
      float y[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        // 0x4B0000qq is the float 2^23 + q (PRMT, no I2F)
        const float big = kk_bits2f(kk_byte_perm(e < 4 ? q0 : q1, 0x4B000000u, 0x7440u | (uint32_t)(e & 3)));
        const float prod = FAST ? kk_fma(dsc, big, dsc2) : __fmul_rn(dsc, __fsub_rn(big, 8388608.0f));
        y[e] = __fsub_rn(prod, dmn);
      }
      store16_all(D, dst_off + (uint64_t)(b0 + k) * 512u + (uint32_t)lane * 16u,
                  make_uint4(pack2<F16>(y[0], y[1]), pack2<F16>(y[2], y[3]), pack2<F16>(y[4], y[5]), pack2<F16>(y[6], y[7])));
    }
  }
}

template <bool F16, bool ALIGNED, bool Q5>
KK_DQ_DEV void q4k_quad(const Dsts& D, uint32_t pay, uint32_t b0, uint32_t nb, uint64_t dst_off, int lane) {
  // --- decode: lane -> (block b0 + min(lane>>3, nb-1), sub-block lane&7)
  const uint32_t hb = min((uint32_t)(lane >> 3), nb - 1);
  const uint32_t hblk = pay + (b0 + hb) * (Q5 ? 176u : KK_Q4K_BLOCK_BYTES);
  uint32_t h0, s0, s1, s2;
  if (ALIGNED) {
    const uint4 h = lds128(hblk);
    h0 = h.x; s0 = h.y; s1 = h.z; s2 = h.w;
  } else {
    h0 = lds32_bytes(hblk); s0 = lds32_bytes(hblk + 4); s1 = lds32_bytes(hblk + 8); s2 = lds32_bytes(hblk + 12);
  }
  const float d = kk_h2f(h0 & 0xFFFFu);
  const float dmin = kk_h2f(h0 >> 16);
  const int j = lane & 7, sh = (j & 3) * 8;
  const uint32_t b_lo = (s0 >> sh) & 0xFFu, b_mid = (s1 >> sh) & 0xFFu, b_hi = (s2 >> sh) & 0xFFu;
  const uint32_t sc = (j < 4) ? (b_lo & 63u) : ((b_hi & 0xFu) | ((b_lo >> 6) << 4));
  const uint32_t mn = (j < 4) ? (b_mid & 63u) : ((b_hi >> 4) | ((b_mid >> 6) << 4));
  const float dsc_j = __fmul_rn(d, (float)sc);
  const float dmn_j = __fmul_rn(dmin, (float)mn);
  const float dsc_c = __fmul_rn(dsc_j, -8388608.0f);
  // fast form iff every scale of the quad is finite and >= +0: then c is -|x| or -0, i.e. its bits lie in [0x80000000, 0xFF800000)
  const bool ok = (kk_f2bits(dsc_c) - 0x80000000u) < 0x7F800000u;
  if (kk_all(ok)) q4k_expand<F16, ALIGNED, true, Q5>(D, pay, b0, nb, dst_off, lane, dsc_j, dsc_c, dmn_j);
  else q4k_expand<F16, ALIGNED, false, Q5>(D, pay, b0, nb, dst_off, lane, dsc_j, dsc_c, dmn_j);
}

template <bool F16>
KK_DQ_DEV void consume_q4k(const Dsts& D, uint32_t pay, uint32_t nblk, uint64_t dst_off, int cwarp, int lane) {
  const bool al = (pay & 15u) == 0;  // 144-byte blocks keep the tile's alignment class
  for (uint32_t b0 = (uint32_t)cwarp * 4u; b0 < nblk; b0 += kConsumerWarps * 4u) {
    const uint32_t nb = min(4u, nblk - b0);
    if (al) q4k_quad<F16, true, false>(D, pay, b0, nb, dst_off, lane);
    else q4k_quad<F16, false, false>(D, pay, b0, nb, dst_off, lane);
  }
}
// Q5_K through the same quads (round 1 gave it one block per warp iteration with ten shared loads per lane, the slowest
// dequantiser; the header decode is now amortised over four blocks and handed out by shuffles like Q4_K's)
template <bool F16>
KK_DQ_DEV void consume_q5k(const Dsts& D, uint32_t pay, uint32_t nblk, uint64_t dst_off, int cwarp, int lane) {
  const bool al = (pay & 15u) == 0;  // 176-byte blocks keep the tile's alignment class
  for (uint32_t b0 = (uint32_t)cwarp * 4u; b0 < nblk; b0 += kConsumerWarps * 4u) {
    const uint32_t nb = min(4u, nblk - b0);
    if (al) q4k_quad<F16, true, true>(D, pay, b0, nb, dst_off, lane);
    else q4k_quad<F16, false, true>(D, pay, b0, nb, dst_off, lane);
  }
}

