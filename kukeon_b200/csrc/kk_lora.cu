// kk_lora_merge_kernel: the LoRA merge of kk_load_adapter (in place) and kk_derive_adapter (out of place) over one device's pool (the arithmetic
// and the tile walk: kk_lora.cuh).  One CTA per tile of every target in the table; every target element is read from `src` and written to `dst`
// once, A and B come from L2 through shared memory.  src and dst are not __restrict__: in place they are the same pool.
#include <cuda_runtime.h>

#include "kk_kernels.cuh"
#include "kk_lora.cuh"

namespace kk {

namespace {

__global__ void __launch_bounds__(KK_LORA_THREADS) kk_lora_merge_kernel(const KKLoraTarget* __restrict__ T, uint32_t n_targets,
                                                                        const float* __restrict__ ad, const uint8_t* src, uint8_t* dst) {
  __shared__ float Bs[KK_LORA_TILE_R * KK_LORA_BS_LD];
  __shared__ __align__(16) float As[KK_LORA_KSTEP * KK_LORA_TILE_C];
  const uint32_t tile = blockIdx.x, tid = threadIdx.x;
  const KKLoraTarget t = T[kk_lora_find(T, n_targets, tile)];
  const KKLoraTile g = kk_lora_tile(t, tile);
  float acc[KK_LORA_TM][KK_LORA_TN];
  KK_LORA_UNROLL
  for (uint32_t ii = 0; ii < KK_LORA_TM; ++ii)
    KK_LORA_UNROLL
    for (uint32_t jj = 0; jj < KK_LORA_TN; ++jj) acc[ii][jj] = 0.0f;
  for (uint32_t k0 = 0; k0 < t.r; k0 += KK_LORA_KSTEP) {
    if (k0) __syncthreads();  // every thread is done with the previous step's values
    kk_lora_stage(t, g, k0, ad, Bs, As, tid);
    __syncthreads();
    const uint32_t kn = t.r - k0 < KK_LORA_KSTEP ? t.r - k0 : KK_LORA_KSTEP;
    kk_lora_fma_step(Bs, As, kn, tid, acc);
  }
  kk_lora_store(t, g, src, dst, tid, acc);
}

}  // namespace

cudaError_t launch_lora_merge(const KKLoraTarget* targets, uint32_t n_targets, uint32_t n_tiles, const float* adapter, const uint8_t* src,
                              uint8_t* dst, cudaStream_t stream) {
  if (n_tiles == 0) return cudaSuccess;
  kk_lora_merge_kernel<<<n_tiles, KK_LORA_THREADS, 0, stream>>>(targets, n_targets, adapter, src, dst);
  return cudaGetLastError();
}

}  // namespace kk
