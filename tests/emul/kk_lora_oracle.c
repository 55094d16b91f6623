/* C oracle of the LoRA merge (kk_load_adapter): the documented arithmetic written out as plain loops, independently of the kernel's header.
 * Widening and rounding go through the F16C instructions for f16 and integer arithmetic for bf16.  Built without fast-math and without FP
 * contraction (tests/lora_fixtures.py), so fmaf is the C library's correctly rounded fused multiply-add and subnormals survive. */
#include <immintrin.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

enum { OUT_BF16 = 0, OUT_F16 = 1, OUT_F32 = 2 };

static float widen(const uint8_t* p, uint32_t out) {
  if (out == OUT_F32) {
    float f;
    memcpy(&f, p, 4);
    return f;
  }
  uint16_t h;
  memcpy(&h, p, 2);
  if (out == OUT_F16) return _cvtsh_ss(h);
  uint32_t u = (uint32_t)h << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}

static void narrow(uint8_t* p, float v, uint32_t out) {
  if (out == OUT_F32) {
    uint32_t u;
    memcpy(&u, &v, 4);
    if (isnan(v)) u = 0x7FFFFFFFu;
    memcpy(p, &u, 4);
    return;
  }
  uint16_t h;
  if (isnan(v)) {
    h = 0x7FFF;
  } else if (out == OUT_F16) {
    h = _cvtss_sh(v, _MM_FROUND_TO_NEAREST_INT);
  } else {
    uint32_t u;
    memcpy(&u, &v, 4);
    const uint32_t rest = u & 0xFFFFu, half = 0x8000u;
    uint32_t hi = u >> 16;
    if (rest > half || (rest == half && (hi & 1u))) hi += 1u;  /* nearest, ties to even; a carry into the exponent gives inf */
    h = (uint16_t)hi;
  }
  memcpy(p, &h, 2);
}

/* Merge one target into `pool`: the [rows, cols] part of a [R, a_ld] tensor that starts at (row0, col0), stored row-major at byte w_off.
 * A is [r, a_ld] and B is [R, r], both fp32. */
void kk_lora_oracle_merge(uint8_t* pool, uint64_t w_off, uint32_t rows, uint32_t cols, uint32_t row0, uint32_t col0, const float* A, uint32_t a_ld,
                          const float* B, uint32_t r, float s, uint32_t out) {
  const uint32_t es = out == OUT_F32 ? 4u : 2u;
  for (uint32_t i = 0; i < rows; ++i)
    for (uint32_t j = 0; j < cols; ++j) {
      float acc = 0.0f;
      for (uint32_t k = 0; k < r; ++k) acc = fmaf(B[(uint64_t)(row0 + i) * r + k], A[(uint64_t)k * a_ld + col0 + j], acc);
      uint8_t* e = pool + w_off + ((uint64_t)i * cols + j) * es;
      narrow(e, fmaf(s, acc, widen(e, out)), out);
    }
}
