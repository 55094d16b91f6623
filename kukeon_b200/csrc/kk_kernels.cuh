// Launch interface of the sm_90a kernels (implemented in kk_kernels.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kk_ops.h"

struct KKLoraTarget;  // kk_lora.cuh

namespace kk {

struct ConvertLaunch {
  const uint8_t* src;        // device (or mapped pinned-host) base of the staged bytes
  const KKSeg* segs;         // device pointer to this launch's segment table
  uint32_t n_segs;
  uint32_t n_tiles;
  uint32_t n_dst;            // 1 = local pool only; >1 = fused fan-out to peer pools
  uint32_t flags;            // KK_LAUNCH_*
  uint8_t* dst[KK_MAX_DST];  // pool bases (dst[0] is the local pool); multimem VA when NVLS
  uint8_t* xdst[KK_MAX_DST]; // KK_OP_ROWSPLIT only: pool of every rank, indexed by rank (all-to-all destinations)
  uint32_t n_xdst;
  uint32_t pad_;
  // Tile-scheduling counters, required: two zeroed uint32 in device memory, private to the STREAM this launch is enqueued on ([0] next batch
  // of tiles, [1] CTAs finished; the last CTA zeroes both again, so consecutive launches on one stream share them).
  uint32_t* sched;
};

// KK_LAUNCH_* flag values: kk_ops.h

// Max segments one launch may carry (tile_begin[] is cached in shared memory).
constexpr uint32_t kMaxSegsPerLaunch = 4096;

// Enqueue the convert / fan-out kernel. Returns the CUDA error (no sync).
cudaError_t launch_convert(const ConvertLaunch& L, int sm_count, cudaStream_t stream);

// out[0] += checksum of [p, p+nbytes) (see kukeon_gpuload.h kk_checksum). p must be 8-byte aligned.
cudaError_t launch_checksum(const uint8_t* p, uint64_t nbytes, unsigned long long* out, int sm_count,
                            cudaStream_t stream);

// Plain ld.global.v4 / st.global.v4 copy, kept for A/B measurement against the TMA path.
cudaError_t launch_ldg_copy(const uint8_t* src, uint8_t* dst, uint64_t nbytes, int sm_count, cudaStream_t stream);

// Store-only probe (no reads): nbytes and dst multiples of 16.
cudaError_t launch_fill(uint8_t* dst, uint64_t nbytes, int sm_count, cudaStream_t stream);

// One-time per-device function attribute setup (dynamic shared memory opt-in).
cudaError_t kernels_init_device();

// LoRA merge (kk_lora.cu): one CTA per tile of the n_targets targets (device table, sorted by tile_begin), reading the target elements of
// pool `src` and writing them merged to the same offsets of pool `dst` (src == dst: in place), with every A and B in `adapter` as fp32.
// Writes nothing outside the targets.  n_tiles < 2^31.
cudaError_t launch_lora_merge(const KKLoraTarget* targets, uint32_t n_targets, uint32_t n_tiles, const float* adapter, const uint8_t* src,
                              uint8_t* dst, cudaStream_t stream);

}  // namespace kk
