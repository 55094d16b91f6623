// LoRA merge (kk_load_adapter, kk_derive_adapter): W += s * B.A over finished pool tensors, shared by kk_lora_merge_kernel (kk_lora.cu) and its CPU
// replay (tests/emul/kk_lora_emul.cpp).  Everything here is KK_HD and touches memory only through the pointers it is given.
//
// Per element (i, j) of a target, in the coordinates of the full tensor:
//   acc = 0.0f;  for k = 0 .. r-1: acc = fmaf(B[i][k], A[k][j], acc)     (strictly this order)
//   v   = fmaf(s, acc, w)                                                  (w: the pool element widened to fp32)
//   out = v rounded to nearest even into the pool dtype (overflow -> inf), any NaN -> 0x7FFF / 0x7FFFFFFF
// The walk: a target is cut into KK_LORA_TILE_R x KK_LORA_TILE_C tiles of W, one CTA of KK_LORA_THREADS threads per tile.  The CTA stages
// the tile's B rows and A columns in shared memory, KK_LORA_KSTEP values of k at a time, and every thread keeps KK_LORA_TM x KK_LORA_TN
// accumulators in registers, so each staged A or B value serves KK_LORA_TM or KK_LORA_TN outputs.  FFMA only: a tensor-core MMA has no
// defined summation order, and the rule above needs one.
#pragma once
#include <stdint.h>
#include <string.h>

#include "kk_ops.h"

#ifdef __CUDACC__
#define KK_LORA_UNROLL _Pragma("unroll")
#else
#define KK_LORA_UNROLL
#endif

#define KK_LORA_TILE_R 64u
#define KK_LORA_TILE_C 128u
#define KK_LORA_THREADS 256u
#define KK_LORA_TM 4u      // rows per thread
#define KK_LORA_TN 8u      // columns per thread: one 16-byte vector of a 16-bit pool, two of an f32 pool
#define KK_LORA_KSTEP 32u  // values of k staged per step
#define KK_LORA_BS_LD (KK_LORA_KSTEP + 1u)  // padded row of the staged B: the 16 row groups of a warp read 16 different banks
#define KK_LORA_MAX_R 256u

// Pool dtype of a target (KKLoraTarget::out).
#define KK_LORA_BF16 0u
#define KK_LORA_F16 1u
#define KK_LORA_F32 2u

// One target tensor of a merge launch.  The adapter buffer holds every A ([r, a_ld]) and B ([R, r]) widened to fp32.
struct KKLoraTarget {
  uint64_t w_off;       // pool byte offset of the tensor (of its slice under SCATTER), row-major [rows, cols]
  uint64_t a_off;       // index of A[0][0] in the adapter buffer (floats)
  uint64_t b_off;       // index of B[0][0]
  uint32_t rows, cols;  // the pool's part of the tensor
  uint32_t row0, col0;  // where that part starts in the full tensor (SCATTER slice_begin along dim 0 or 1)
  uint32_t a_ld;        // columns of the full tensor: the row stride of A
  uint32_t r;           // rank, 1..KK_LORA_MAX_R
  float s;              // scaling
  uint32_t out;         // KK_LORA_BF16 / KK_LORA_F16 / KK_LORA_F32
  uint32_t tile_begin;  // first tile of this target in the launch (the table is sorted by it)
  uint32_t tiles_c;     // column tiles of this target
};
#ifdef __cplusplus
static_assert(sizeof(KKLoraTarget) == 64, "KKLoraTarget layout is shared with the device");
#endif

struct alignas(16) KKLoraVec {
  uint32_t w[4];
};

static inline KK_HD uint32_t kk_lora_tiles(uint32_t rows, uint32_t cols) {
  return ((rows + KK_LORA_TILE_R - 1) / KK_LORA_TILE_R) * ((cols + KK_LORA_TILE_C - 1) / KK_LORA_TILE_C);
}

static inline KK_HD uint32_t kk_lora_f2u(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
}
static inline KK_HD float kk_lora_u2f(uint32_t u) {
  float f;
  memcpy(&f, &u, 4);
  return f;
}

// Exact widenings.
static inline KK_HD float kk_lora_bf16_f32(uint16_t h) { return kk_lora_u2f((uint32_t)h << 16); }
static inline KK_HD float kk_lora_f16_f32(uint16_t h) {
  const uint32_t s = (uint32_t)(h & 0x8000u) << 16, e = (h >> 10) & 0x1Fu, m = h & 0x3FFu;
  if (e == 0x1Fu) return kk_lora_u2f(s | 0x7F800000u | (m << 13));
  if (e == 0) return kk_lora_u2f(s | kk_lora_f2u((float)m * 5.9604644775390625e-8f));  // m * 2^-24: exact, a normal fp32
  return kk_lora_u2f(s | ((e + 112u) << 23) | (m << 13));
}

// Round to nearest even; NaN -> 0x7FFF.
static inline KK_HD uint16_t kk_lora_f32_bf16(float f) {
  uint32_t x = kk_lora_f2u(f);
  if ((x & 0x7FFFFFFFu) > 0x7F800000u) return 0x7FFFu;
  x += 0x7FFFu + ((x >> 16) & 1u);
  return (uint16_t)(x >> 16);
}
static inline KK_HD uint16_t kk_lora_f32_f16(float f) {
  uint32_t x = kk_lora_f2u(f);
  const uint32_t sign = (x >> 16) & 0x8000u;
  x &= 0x7FFFFFFFu;
  if (x > 0x7F800000u) return 0x7FFFu;
  uint32_t o;
  if (x >= 0x47800000u) {  // >= 65536: inf
    o = 0x7C00u;
  } else if (x < 0x38800000u) {  // below the smallest normal f16: one fp32 add lines the 10 mantissa bits up at the bottom, rounding to nearest even
    const float magic = kk_lora_u2f(0x3F000000u);  // 0.5
    o = kk_lora_f2u(kk_lora_u2f(x) + magic) - 0x3F000000u;
  } else {  // normal (a carry out of the mantissa rounds [65520, 65536) to inf)
    x += 0xC8000FFFu + ((x >> 13) & 1u);
    o = x >> 13;
  }
  return (uint16_t)(o | sign);
}

static inline KK_HD float kk_lora_fma(float a, float b, float c) {
#ifdef __CUDA_ARCH__
  return __fmaf_rn(a, b, c);
#else
  return __builtin_fmaf(a, b, c);
#endif
}

// The merged element: w widened, v = fmaf(s, acc, w), rounded into the pool dtype.
static inline KK_HD uint16_t kk_lora_merge16(uint16_t w, float acc, float s, uint32_t out) {
  if (out == KK_LORA_F16) return kk_lora_f32_f16(kk_lora_fma(s, acc, kk_lora_f16_f32(w)));
  return kk_lora_f32_bf16(kk_lora_fma(s, acc, kk_lora_bf16_f32(w)));
}
static inline KK_HD uint32_t kk_lora_merge32(uint32_t w, float acc, float s) {
  const float v = kk_lora_fma(s, acc, kk_lora_u2f(w));
  return v != v ? 0x7FFFFFFFu : kk_lora_f2u(v);
}

// The target that owns launch tile `tile` (table sorted by tile_begin, tile inside the launch).
static inline KK_HD uint32_t kk_lora_find(const KKLoraTarget* T, uint32_t n, uint32_t tile) {
  uint32_t lo = 0, hi = n;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) / 2;
    if (T[mid].tile_begin <= tile) lo = mid;
    else hi = mid;
  }
  return lo;
}

// Tile (ti, tj) of target t: first row and column in the pool's part.
struct KKLoraTile {
  uint32_t i0, j0;
};
static inline KK_HD KKLoraTile kk_lora_tile(const KKLoraTarget& t, uint32_t tile) {
  const uint32_t k = tile - t.tile_begin;
  return {(k / t.tiles_c) * KK_LORA_TILE_R, (k % t.tiles_c) * KK_LORA_TILE_C};
}

// Step 1 of each k step, thread `tid`: stage its share of B[i0 .., k0 ..] into Bs[KK_LORA_TILE_R][KK_LORA_BS_LD] and of A[k0 .., j0 ..] into
// As[KK_LORA_KSTEP][KK_LORA_TILE_C]; values outside the target or past r are staged as 0 and never summed.
static inline KK_HD void kk_lora_stage(const KKLoraTarget& t, KKLoraTile g, uint32_t k0, const float* ad, float* Bs, float* As, uint32_t tid) {
  KK_LORA_UNROLL
  for (uint32_t q = 0; q < KK_LORA_TILE_R * KK_LORA_KSTEP / KK_LORA_THREADS; ++q) {
    const uint32_t idx = tid + q * KK_LORA_THREADS, row = idx / KK_LORA_KSTEP, kk = idx % KK_LORA_KSTEP;
    const uint32_t i = g.i0 + row, k = k0 + kk;
    Bs[row * KK_LORA_BS_LD + kk] = (i < t.rows && k < t.r) ? ad[t.b_off + (uint64_t)(t.row0 + i) * t.r + k] : 0.0f;
  }
  KK_LORA_UNROLL
  for (uint32_t q = 0; q < KK_LORA_KSTEP * KK_LORA_TILE_C / KK_LORA_THREADS; ++q) {
    const uint32_t idx = tid + q * KK_LORA_THREADS, kk = idx / KK_LORA_TILE_C, col = idx % KK_LORA_TILE_C;
    const uint32_t j = g.j0 + col, k = k0 + kk;
    As[kk * KK_LORA_TILE_C + col] = (j < t.cols && k < t.r) ? ad[t.a_off + (uint64_t)k * t.a_ld + t.col0 + j] : 0.0f;
  }
}

// Step 2, thread `tid`: the kn staged values of k, in order, into its accumulators.
static inline KK_HD void kk_lora_fma_step(const float* Bs, const float* As, uint32_t kn, uint32_t tid, float acc[KK_LORA_TM][KK_LORA_TN]) {
  const uint32_t ty = tid / (KK_LORA_TILE_C / KK_LORA_TN), tx = tid % (KK_LORA_TILE_C / KK_LORA_TN);
  for (uint32_t kk = 0; kk < kn; ++kk) {
    float b[KK_LORA_TM], a[KK_LORA_TN];
    KK_LORA_UNROLL
    for (uint32_t ii = 0; ii < KK_LORA_TM; ++ii) b[ii] = Bs[(ty * KK_LORA_TM + ii) * KK_LORA_BS_LD + kk];
    KK_LORA_UNROLL
    for (uint32_t jj = 0; jj < KK_LORA_TN; ++jj) a[jj] = As[kk * KK_LORA_TILE_C + tx * KK_LORA_TN + jj];
    KK_LORA_UNROLL
    for (uint32_t ii = 0; ii < KK_LORA_TM; ++ii)
      KK_LORA_UNROLL
      for (uint32_t jj = 0; jj < KK_LORA_TN; ++jj) acc[ii][jj] = kk_lora_fma(b[ii], a[jj], acc[ii][jj]);
  }
}

// Step 3, thread `tid`: read its outputs' elements from the pool `src`, merge them and write them to the same offsets of the pool `dst`.  Whole
// 16-byte vectors where the row has them, single elements at the right edge and in rows that are not 16-byte multiples; nothing outside the
// target.  src == dst merges in place (kk_load_adapter), src != dst out of place (kk_derive_adapter): each element is read and then written by
// the same thread, so the two may alias.
static inline KK_HD void kk_lora_store(const KKLoraTarget& t, KKLoraTile g, const uint8_t* src, uint8_t* dst, uint32_t tid,
                                       const float acc[KK_LORA_TM][KK_LORA_TN]) {
  const uint32_t ty = tid / (KK_LORA_TILE_C / KK_LORA_TN), tx = tid % (KK_LORA_TILE_C / KK_LORA_TN);
  const uint32_t es = t.out == KK_LORA_F32 ? 4u : 2u;
  const uint32_t j0 = g.j0 + tx * KK_LORA_TN;
  if (j0 >= t.cols) return;
  const bool vec = j0 + KK_LORA_TN <= t.cols && ((uint64_t)t.cols * es) % 16 == 0;
  KK_LORA_UNROLL
  for (uint32_t ii = 0; ii < KK_LORA_TM; ++ii) {
    const uint32_t i = g.i0 + ty * KK_LORA_TM + ii;
    if (i >= t.rows) break;
    const uint64_t at = t.w_off + ((uint64_t)i * t.cols + j0) * es;
    const uint8_t* in = src + at;
    uint8_t* row = dst + at;
    if (vec && es == 2) {
      KKLoraVec v = *(const KKLoraVec*)in;
      KK_LORA_UNROLL
      for (uint32_t q = 0; q < 4; ++q) {
        const uint32_t lo = kk_lora_merge16((uint16_t)(v.w[q] & 0xFFFFu), acc[ii][2 * q], t.s, t.out);
        const uint32_t hi = kk_lora_merge16((uint16_t)(v.w[q] >> 16), acc[ii][2 * q + 1], t.s, t.out);
        v.w[q] = lo | (hi << 16);
      }
      *(KKLoraVec*)row = v;
    } else if (vec) {
      KK_LORA_UNROLL
      for (uint32_t h = 0; h < 2; ++h) {
        KKLoraVec v = *(const KKLoraVec*)(in + 16 * h);
        KK_LORA_UNROLL
        for (uint32_t q = 0; q < 4; ++q) v.w[q] = kk_lora_merge32(v.w[q], acc[ii][4 * h + q], t.s);
        *(KKLoraVec*)(row + 16 * h) = v;
      }
    } else {
      for (uint32_t jj = 0; jj < KK_LORA_TN && j0 + jj < t.cols; ++jj) {
        if (es == 2) {
          uint16_t w;
          memcpy(&w, in + jj * 2, 2);
          w = kk_lora_merge16(w, acc[ii][jj], t.s, t.out);
          memcpy(row + jj * 2, &w, 2);
        } else {
          uint32_t w;
          memcpy(&w, in + jj * 4, 4);
          w = kk_lora_merge32(w, acc[ii][jj], t.s);
          memcpy(row + jj * 4, &w, 4);
        }
      }
    }
  }
}

// Step 3 in place: src == dst == pool.
static inline KK_HD void kk_lora_store(const KKLoraTarget& t, KKLoraTile g, uint8_t* pool, uint32_t tid, const float acc[KK_LORA_TM][KK_LORA_TN]) {
  kk_lora_store(t, g, pool, pool, tid, acc);
}
