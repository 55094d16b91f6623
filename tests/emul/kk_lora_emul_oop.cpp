// CPU replay of the out-of-place launch of kk_lora_merge_kernel (kk_derive_adapter; test infrastructure): as kk_lora_emul.cpp, the launch's
// CTA grid played tile by tile through kukeon_b200/csrc/kk_lora.cuh, with the target elements read from `src` and written to `dst` (which may
// be `src`).
#include <stdint.h>

#include <vector>

#include "../../kukeon_b200/csrc/kk_lora.cuh"

extern "C" int kk_lora_emul_launch_oop(const KKLoraTarget* T, uint32_t n_targets, uint32_t n_tiles, const float* ad, const uint8_t* src, uint8_t* dst) {
  if (n_targets == 0) return n_tiles == 0 ? 0 : -1;
  std::vector<float> Bs(KK_LORA_TILE_R * KK_LORA_BS_LD), As(KK_LORA_KSTEP * KK_LORA_TILE_C);
  std::vector<float> acc(KK_LORA_THREADS * KK_LORA_TM * KK_LORA_TN);
  auto acc_of = [&](uint32_t tid) { return reinterpret_cast<float(*)[KK_LORA_TN]>(acc.data() + tid * KK_LORA_TM * KK_LORA_TN); };
  for (uint32_t tile = 0; tile < n_tiles; ++tile) {
    const KKLoraTarget t = T[kk_lora_find(T, n_targets, tile)];
    if (tile < t.tile_begin) return -1;
    const KKLoraTile g = kk_lora_tile(t, tile);
    for (float& a : acc) a = 0.0f;
    for (uint32_t k0 = 0; k0 < t.r; k0 += KK_LORA_KSTEP) {
      for (uint32_t tid = 0; tid < KK_LORA_THREADS; ++tid) kk_lora_stage(t, g, k0, ad, Bs.data(), As.data(), tid);
      const uint32_t kn = t.r - k0 < KK_LORA_KSTEP ? t.r - k0 : KK_LORA_KSTEP;
      for (uint32_t tid = 0; tid < KK_LORA_THREADS; ++tid) kk_lora_fma_step(Bs.data(), As.data(), kn, tid, acc_of(tid));
    }
    for (uint32_t tid = 0; tid < KK_LORA_THREADS; ++tid) kk_lora_store(t, g, src, dst, tid, acc_of(tid));
  }
  return 0;
}
