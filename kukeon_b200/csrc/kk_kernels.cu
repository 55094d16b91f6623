// sm_90a kernels of the weight loader: one persistent, warp-specialised convert / fan-out kernel
// plus a checksum kernel.  No tensor cores — the path has no contraction; it is HBM / NVLink bound.
//
// kk_convert_kernel:
//   warp 0 (one elected lane) = TMA producer. It walks this CTA's tiles, resolves tile -> segment,
//     publishes a TileDesc and pulls the tile's source bytes into a 4-stage shared-memory ring with
//     cp.async.bulk (UBLKCP) completing on an mbarrier.
//   warps 1..16 = consumers. Depending on the segment op they
//       COPY, aligned     : one lane fires cp.async.bulk shared->global stores, one per destination pool
//                           (local pool + peer-mapped pools: the fused fan-out), no register traffic;
//       F32/F16 -> BF16   : ld.shared.v4, cvt.rn.bf16x2.f32, st.global.v4 (16 B per lane, coalesced);
//       Q4_K -> BF16      : one warp per 256-weight super-block; the 8 (scale,min) pairs are decoded once
//                           and handed to the lanes with __shfl_sync; nibbles become floats with a PRMT
//                           + FADD magic-number trick; every lane stores 16 B of bf16;
//       other GGUF quants : every other block type, one lane per 8 weights (kk_dequant.cuh);
//       2-D transposes    : 8-row tiles staged by bulk copies, thread = column, one 16-byte store per column (GPT-2 Conv1D weights).
//   Every output vector is stored to n_dst pools; dst[1..] are NVLink peer mappings, so conversion and
//   broadcast are ONE kernel and the source bytes are read from HBM exactly once.
//   The kernel keeps the tile scheduling and the stage protocol; the segment lookup (kk_tile_seg), the tile (kk_make_tile), its copies
//   (kk_load_tile), its bulk stores (kk_store_tile) and the consumer dispatch (kk_consume_tile) are the functions tests/emul plays on the CPU.
//
// kk_convert_f16_kernel: the same kernel instantiated for IEEE fp16 output (KK_LOAD_F16 models; launch_convert picks it from
//   KK_LAUNCH_F16).  Every pack is cvt.rn.f16x2.f32 instead of cvt.rn.bf16x2.f32, the 16-bit casts take bf16 in, and FP8 stores the
//   hardware's f16x2 pair as it is.  Two kernels rather than a branch: neither reads the flag, and the bf16 kernel's code is unchanged.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "kk_iq_grids.h"
#include "kk_kernels.cuh"
#include "kk_tile.h"

namespace kk {

namespace {

constexpr int kStages = 4;
constexpr int kConsumerWarps = KK_CONSUMER_WARPS;
constexpr int kConsumerThreads = kConsumerWarps * 32;
constexpr int kThreads = 32 + kConsumerThreads;  // 544
constexpr uint32_t kStageBytes = KK_TILE_SRC_BYTES + KK_STAGE_PAD;

using TileDesc = KKTileDesc;  // kk_tile.h: the producer computes every tile with kk_make_tile, the function tests/emul replays launches through
static_assert(sizeof(TileDesc) == 64, "TileDesc");

constexpr uint32_t kSmemFixed = kStages * kStageBytes + kStages * sizeof(TileDesc) + 2 * kStages * 8;

// ---- PTX wrappers ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "KK_WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra KK_DONE_%=;\n\t"
      "bra KK_WAIT_%=;\n\t"
      "KK_DONE_%=:\n\t"
      "}" ::"r"(bar), "r"(parity)
      : "memory");
}
// global -> shared bulk copy (TMA, non-tensor form). src, dst and bytes are multiples of 16.
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// shared -> global bulk copy.
__device__ __forceinline__ void bulk_s2g(void* dst, uint32_t src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src_smem), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Loads from the staged tile are PLAIN C++ loads (the compiler infers ld.shared from the cvta intrinsic), not volatile asm: the compiler may then
// hoist the loads of the next block above the arithmetic and the global store of the previous one — the stores below carry no "memory" clobber
// for the same reason — which is where a warp's instruction-level parallelism comes from (with volatile asm every block's load -> math -> store
// chain ran strictly after the previous block's: Q3_K sat at 0.54 of the copy peak, latency-bound with 4 warps per scheduler).  Ordering against
// the pipeline is kept by the "memory" clobbers of mbar_wait (acquire of the stage), mbar_arrive (release) and the named barrier.
template <typename T>
__device__ __forceinline__ T lds_plain(uint32_t a) {
  return *reinterpret_cast<const T*>(__cvta_shared_to_generic((size_t)a));
}
__device__ __forceinline__ uint4 lds128(uint32_t a) { return lds_plain<uint4>(a); }
__device__ __forceinline__ uint2 lds64(uint32_t a) { return lds_plain<uint2>(a); }
__device__ __forceinline__ uint32_t lds8(uint32_t a) { return lds_plain<uint8_t>(a); }
__device__ __forceinline__ void stg128(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w));  // no "memory" clobber: see lds_plain
}
__device__ __forceinline__ void stmm128(void* p, const uint4& v) {  // NVLS multicast store
  asm volatile("multimem.st.weak.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(__uint_as_float(v.x)),
               "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)), "f"(__uint_as_float(v.w))
               : "memory");
}
__device__ __forceinline__ void named_bar_consumers() { asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory"); }
__device__ __forceinline__ void rowsplit_store1(const ConvertLaunch& L, uint32_t j, uint64_t off, uint8_t v) { L.xdst[j][off] = v; }
__device__ __forceinline__ void rowsplit_store_bulk(const ConvertLaunch& L, uint32_t j, uint64_t off, uint32_t src_smem, uint32_t bytes) {
  bulk_s2g(L.xdst[j] + off, src_smem, bytes);
}
// A stage as the producer fills it: its shared-memory address and the mbarrier its copies complete on.
struct StageLoad {
  const uint8_t* src;
  uint32_t smem, bar;
};
__device__ __forceinline__ void bulk_load(const StageLoad& S, uint32_t stage_off, uint64_t g_off, uint32_t bytes) {
  bulk_g2s(S.smem + stage_off, S.src + g_off, bytes, S.bar);
}

// Two floats -> packed bf16x2 (a in the low half), round-to-nearest-even; NaN -> 0x7FFF.
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
// Two floats -> packed f16x2 (a in the low half), round-to-nearest-even, overflow -> +-inf, fp16 subnormals kept; NaN -> 0x7FFF.
__device__ __forceinline__ uint32_t pack_f16x2(float a, float b) {
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}

struct Dsts {
  uint8_t* p[KK_MAX_DST];
  uint32_t n;
  bool multimem;
  bool single;  // n == 1 and not multimem
};

// 16-byte store of one output vector to every destination pool.
__device__ __forceinline__ void store16_all(const Dsts& D, uint64_t off, const uint4& v) {
  if (D.single) {  // the common N = 1 case: no per-store predicate ladder
    stg128(D.p[0] + off, v);
    return;
  }
  if (D.multimem) {
    stmm128(D.p[0] + off, v);
    return;
  }
#pragma unroll
  for (int d = 0; d < KK_MAX_DST; ++d)
    if (d < (int)D.n) stg128(D.p[d] + off, v);
}
// 8-byte store of half an output vector (the aligned F32 -> bf16 cast: 4 elements per thread) to every destination pool
__device__ __forceinline__ void store8_all(const Dsts& D, uint64_t off, uint32_t lo, uint32_t hi) {
  if (D.multimem) {
    asm volatile("multimem.st.weak.global.v2.f32 [%0], {%1,%2};" ::"l"(D.p[0] + off), "f"(__uint_as_float(lo)), "f"(__uint_as_float(hi)) : "memory");
    return;
  }
#pragma unroll
  for (int d = 0; d < KK_MAX_DST; ++d)
    if (d < (int)D.n) asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" ::"l"(D.p[d] + off), "r"(lo), "r"(hi));
}
// bulk store of `bytes` from the stage to destination pool d
__device__ __forceinline__ void store_bulk(const Dsts& D, int d, uint64_t off, uint32_t src_smem, uint32_t bytes) { bulk_s2g(D.p[d] + off, src_smem, bytes); }
__device__ __forceinline__ void store2_all(const Dsts& D, uint64_t off, uint16_t v) {
  if (D.multimem) {
    // multimem.st has no 8- or 16-bit form: the host only selects KK_LAUNCH_MULTIMEM for plans whose segments never need a
    // sub-4-byte store (kk_loader.cpp plan_allows_multimem), so this is unreachable there.
    return;
  }
#pragma unroll
  for (int d = 0; d < KK_MAX_DST; ++d)
    if (d < (int)D.n) *reinterpret_cast<uint16_t*>(D.p[d] + off) = v;
}
__device__ __forceinline__ void store1_all(const Dsts& D, uint64_t off, uint8_t v) {
  if (D.multimem) return;
#pragma unroll
  for (int d = 0; d < KK_MAX_DST; ++d)
    if (d < (int)D.n) D.p[d][off] = v;
}
__device__ __forceinline__ void store4_all(const Dsts& D, uint64_t off, uint32_t v) {
  if (D.multimem) {
    asm volatile("multimem.st.weak.global.b32 [%0], %1;" ::"l"(D.p[0] + off), "r"(v) : "memory");
    return;
  }
#pragma unroll
  for (int d = 0; d < KK_MAX_DST; ++d)
    if (d < (int)D.n) *reinterpret_cast<uint32_t*>(D.p[d] + off) = v;
}

// ---- consumer bodies ------------------------------------------------------------------------------------------------------------
// Every per-lane consumer function lives in kk_consume_core.cuh (copy, casts, Q4_K) and kk_dequant.cuh (the other block types, FP8,
// 8-row transposes), and the per-tile dispatch between them in kk_consume_tile.cuh, all written against the primitives bound here so
// that tests/emul can compile the same source for the host.
__device__ __forceinline__ uint32_t lds16(uint32_t a) { return lds_plain<uint16_t>(a); }
__device__ __forceinline__ uint32_t lds32(uint32_t a) { return lds_plain<uint32_t>(a); }
__device__ __forceinline__ float kk_h2f(uint32_t h) { return __half2float(__ushort_as_half((unsigned short)h)); }
// two FP8 (low 16 bits of v) -> two fp16, exact (sm_89+ pair conversion)
template <bool E5M2>
__device__ __forceinline__ uint32_t kk_f8x2_to_f16x2(uint32_t v) {
  uint32_t r;
  const unsigned short s = (unsigned short)v;
  if (E5M2) asm("cvt.rn.f16x2.e5m2x2 %0, %1;" : "=r"(r) : "h"(s));
  else asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(r) : "h"(s));
  return r;
}
__device__ __forceinline__ float kk_bits2f(uint32_t u) { return __uint_as_float(u); }
__device__ __forceinline__ float kk_fma(float a, float b, float c) { return __fmaf_rn(a, b, c); }  // one rounding
__device__ __forceinline__ bool kk_all(bool p) { return __all_sync(0xffffffffu, p) != 0; }  // warp vote
__device__ __forceinline__ uint32_t kk_byte_perm(uint32_t a, uint32_t b, uint32_t sel) { return __byte_perm(a, b, sel); }
__device__ __forceinline__ void sts16(uint32_t a, uint32_t v) { asm volatile("st.shared.u16 [%0], %1;" ::"r"(a), "h"((unsigned short)v) : "memory"); }
__device__ __forceinline__ void sts32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ uint32_t kk_ldg8(const uint8_t* p) { return (uint32_t)__ldg(p); }
__device__ __forceinline__ void kk_h2x2f(uint32_t w, float& x, float& y) {
  const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w));
  x = f.x;
  y = f.y;
}
__device__ __forceinline__ uint32_t kk_f2bits(float f) { return __float_as_uint(f); }
__device__ __forceinline__ uint32_t kk_popc(uint32_t u) { return (uint32_t)__popc(u); }
// SHF.R.W: bits [sh, sh + 32) of the 64-bit value hi:lo (sh taken mod 32)
__device__ __forceinline__ uint32_t kk_funnel_r(uint32_t lo, uint32_t hi, uint32_t sh) { return __funnelshift_r(lo, hi, sh); }
// an aligned word whose first byte is payload but whose last 1-3 bytes may lie in the stage's slack behind it (KK_STAGE_PAD): same load
__device__ __forceinline__ uint32_t lds32_slack(uint32_t a) { return lds32(a); }
// i-quant codebooks (33 KB, read through the read-only path; hot entries stay in L1)
__device__ const uint64_t kGridIq2xxs[KK_GRID_IQ2XXS_SIZE] = {KK_GRID_IQ2XXS_VALUES};
__device__ const uint64_t kGridIq2xs[KK_GRID_IQ2XS_SIZE] = {KK_GRID_IQ2XS_VALUES};
__device__ const uint64_t kGridIq2s[KK_GRID_IQ2S_SIZE] = {KK_GRID_IQ2S_VALUES};
__device__ const uint32_t kGridIq3xxs[KK_GRID_IQ3XXS_SIZE] = {KK_GRID_IQ3XXS_VALUES};
__device__ const uint32_t kGridIq3s[KK_GRID_IQ3S_SIZE] = {KK_GRID_IQ3S_VALUES};
__device__ const uint64_t kGridIq1s[KK_GRID_IQ1S_SIZE] = {KK_GRID_IQ1S_VALUES};
__device__ __forceinline__ uint64_t kk_grid_iq2xxs(uint32_t i) { return __ldg(&kGridIq2xxs[i]); }
__device__ __forceinline__ uint64_t kk_grid_iq2xs(uint32_t i) { return __ldg(&kGridIq2xs[i]); }
__device__ __forceinline__ uint64_t kk_grid_iq2s(uint32_t i) { return __ldg(&kGridIq2s[i]); }
__device__ __forceinline__ uint32_t kk_grid_iq3xxs(uint32_t i) { return __ldg(&kGridIq3xxs[i]); }
__device__ __forceinline__ uint32_t kk_grid_iq3s(uint32_t i) { return __ldg(&kGridIq3s[i]); }
__device__ __forceinline__ uint64_t kk_grid_iq1s(uint32_t i) { return __ldg(&kGridIq1s[i]); }
#define KK_DQ_DEV __device__ __forceinline__
#include "kk_consume_tile.cuh"

__device__ __forceinline__ KKSeg load_seg(const KKSeg* p) {
  const uint4* q = reinterpret_cast<const uint4*>(p);
  uint4 a = __ldg(q), b = __ldg(q + 1), c = __ldg(q + 2);
  KKSeg s;
  s.src_off = ((uint64_t)a.y << 32) | a.x;
  s.dst_off = ((uint64_t)a.w << 32) | a.z;
  s.units = ((uint64_t)b.y << 32) | b.x;
  s.op = b.z;
  s.tile_begin = b.w;
  s.p0 = c.x; s.p1 = c.y; s.p2 = c.z; s.p3 = c.w;
  return s;
}

// The kernel body, for either output format (F16: KK_LAUNCH_F16); the two __global__ instantiations follow it.
template <bool F16>
__device__ __forceinline__ void convert_body(const ConvertLaunch& L) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* stage_buf = smem;
  TileDesc* descs = reinterpret_cast<TileDesc*>(smem + kStages * kStageBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes + kStages * sizeof(TileDesc));
  uint32_t* tile_begin = reinterpret_cast<uint32_t*>(smem + kSmemFixed);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + kStages);

  for (uint32_t i = tid; i < L.n_segs; i += kThreads) tile_begin[i] = L.segs[i].tile_begin;
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, kConsumerWarps);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 0) {
    // ===== producer =====
    if (lane == 0) {
      // Tile scheduling.  Static round-robin (tile = blockIdx.x + k * gridDim.x) leaves the SMs unevenly loaded although every CTA gets the same
      // number of tiles: SMs do not all see the same memory at the same cost (L2 partitions, HBM stacks), and the kernel ends with the slowest
      // CTA.  So after its first, static tile a CTA draws batches of kBatch tiles from a global counter; the draw for batch b + 1 is issued while
      // batch b is being produced, so the atomic's round trip is off the critical path even for the copy op.
      constexpr uint32_t kBatch = 2;
      uint32_t cur = 0;
      KKSeg seg = load_seg(L.segs);
      uint32_t it = 0;
      uint32_t tile = blockIdx.x, batch_next = 0, batch_left = 0;
      uint32_t pre = atomicAdd(L.sched, kBatch);
      for (; tile < L.n_tiles; ++it) {
        const uint32_t s = it % kStages, ph = (it / kStages) & 1u;
        mbar_wait(empty0 + 8 * s, ph ^ 1u);
        const uint32_t nxt = kk_tile_seg(tile_begin, L.n_segs, cur, tile);
        if (nxt != cur) { cur = nxt; seg = load_seg(L.segs + cur); }
        KKTileDesc sd;
        KKTileLoad ld;
        kk_make_tile(seg, tile - seg.tile_begin, (uint64_t)(uintptr_t)L.src, L.flags, sd, ld);
        descs[s] = sd;
        if (ld.kind == 0) {
          mbar_arrive(full0 + 8 * s);
        } else {
          mbar_arrive_expect_tx(full0 + 8 * s, ld.tx);
          kk_load_tile(ld, StageLoad{L.src, smem_u32(stage_buf + s * kStageBytes), full0 + 8 * s});
        }
        if (batch_left == 0) {
          batch_next = gridDim.x + pre;
          batch_left = kBatch;
          pre = atomicAdd(L.sched, kBatch);
        }
        tile = batch_next++;
        --batch_left;
      }
      {  // end marker for the consumers, which do not know in advance how many tiles their CTA draws
        const uint32_t s = it % kStages, ph = (it / kStages) & 1u;
        mbar_wait(empty0 + 8 * s, ph ^ 1u);
        descs[s].op = KK_OP_END;
        mbar_arrive(full0 + 8 * s);
      }
      // the last CTA to get here leaves the counters zeroed for the next launch on this stream
      __threadfence();
      if (atomicAdd(L.sched + 1, 1u) == gridDim.x - 1u) {
        L.sched[0] = 0u;
        L.sched[1] = 0u;
        __threadfence();
      }
    }
  } else {
    // ===== consumers =====
    const int cwarp = warp - 1, ctid = tid - 32;
    Dsts D;
#pragma unroll
    for (int i = 0; i < KK_MAX_DST; ++i) D.p[i] = L.dst[i];
    D.n = L.n_dst;
    D.multimem = (L.flags & KK_LAUNCH_MULTIMEM) != 0;
    D.single = (L.n_dst == 1) && !D.multimem;
    int pending = -1;  // stage whose bulk stores may still be reading shared memory (warp 1 lane 0 only)
    for (uint32_t it = 0;; ++it) {
      const uint32_t s = it % kStages, ph = (it / kStages) & 1u;
      mbar_wait(full0 + 8 * s, ph);
      const TileDesc t = descs[s];
      if (t.op == KK_OP_END) break;  // the producer's end marker
      const uint32_t sbase = smem_u32(stage_buf + s * kStageBytes);
      const uint32_t pay = sbase + t.pay_off;
      // Aligned copy (bulk 1) / row-split exchange (bulk 3): warp 0 lane 0 bulk-stores the stage, released once the stores have read it.
      // Two branches, not one: with the kind known in each, the copy path's issuing lane runs straight through (merged, it took two more
      // branches per tile and the bf16 copy stage ran 0.08 % slower on an H100 80GB HBM3 at a 700 W limit).
      if (t.bulk == 1) {
        if (cwarp == 0) {
          if (lane == 0) {
            fence_proxy_async();
            kk_store_tile(D, t, pay, L);
            bulk_commit();
            if (pending >= 0) {
              bulk_wait_read<1>();
              mbar_arrive(empty0 + 8 * pending);
            }
            pending = (int)s;
          }
        } else {
          if (lane == 0) mbar_arrive(empty0 + 8 * s);
        }
        continue;
      }
      if (t.bulk == 3) {
        if (cwarp == 0) {
          if (lane == 0) {
            fence_proxy_async();
            kk_store_tile(D, t, pay, L);
            bulk_commit();
            if (pending >= 0) {
              bulk_wait_read<1>();
              mbar_arrive(empty0 + 8 * pending);
            }
            pending = (int)s;
          }
        } else {
          if (lane == 0) mbar_arrive(empty0 + 8 * s);
        }
        continue;
      }
      if (cwarp == 0 && lane == 0 && pending >= 0) {
        bulk_wait_read<0>();
        mbar_arrive(empty0 + 8 * pending);
        pending = -1;
      }
      kk_consume_tile<F16>(D, t, sbase, pay, L, cwarp, lane, ctid, it);
      __syncwarp();
      if (lane == 0) mbar_arrive(empty0 + 8 * s);
    }
    if (cwarp == 0 && lane == 0) {
      if (pending >= 0) {
        bulk_wait_read<0>();
        mbar_arrive(empty0 + 8 * pending);
      }
      bulk_wait_all();  // all bulk stores globally performed before the CTA retires
    }
  }
}

__global__ void __launch_bounds__(kThreads, 1) kk_convert_kernel(const ConvertLaunch L) { convert_body<false>(L); }
// fp16 output.  Its name must not contain "kk_convert_kernel": tools/sass_budget.py finds the bf16 kernel by that substring.
__global__ void __launch_bounds__(kThreads, 1) kk_convert_f16_kernel(const ConvertLaunch L) { convert_body<true>(L); }

// ---- checksum ---------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t mix64(uint64_t x) {
  x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull;
  x ^= x >> 27; x *= 0x94d049bb133111ebull;
  x ^= x >> 31;
  return x;
}

__global__ void __launch_bounds__(256) kk_checksum_kernel(const uint8_t* __restrict__ p, uint64_t nbytes, unsigned long long* out) {
  const uint64_t nwords = nbytes >> 3;
  const uint64_t* w = reinterpret_cast<const uint64_t*>(p);
  uint64_t acc = 0;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nwords; i += (uint64_t)gridDim.x * blockDim.x)
    acc += mix64(__ldg(w + i) + i * 0x9E3779B97F4A7C15ull);
  if (blockIdx.x == 0 && threadIdx.x == 0 && (nbytes & 7)) {
    uint64_t last = 0;
    for (uint32_t k = 0; k < (nbytes & 7); ++k) last |= (uint64_t)p[(nwords << 3) + k] << (8 * k);
    acc += mix64(last + nwords * 0x9E3779B97F4A7C15ull);
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0 && acc) atomicAdd(out, (unsigned long long)acc);
}

__global__ void __launch_bounds__(256) kk_ldg_copy_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, uint64_t nvec) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + 3 * stride < nvec; i += 4 * stride) {
    uint4 a = __ldcs(src + i), b = __ldcs(src + i + stride), c = __ldcs(src + i + 2 * stride), d = __ldcs(src + i + 3 * stride);
    __stcs(dst + i, a); __stcs(dst + i + stride, b); __stcs(dst + i + 2 * stride, c); __stcs(dst + i + 3 * stride, d);
  }
  for (; i < nvec; i += stride) __stcs(dst + i, __ldcs(src + i));
}

// Store-only probe: what the box's HBM sustains when a kernel does nothing but write (the "HBM-write roofline" of SURVEY.md §8(d)).
__global__ void __launch_bounds__(256) kk_fill_kernel(uint4* __restrict__ dst, uint64_t nvec, uint4 v) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + 3 * stride < nvec; i += 4 * stride) {
    __stcs(dst + i, v); __stcs(dst + i + stride, v); __stcs(dst + i + 2 * stride, v); __stcs(dst + i + 3 * stride, v);
  }
  for (; i < nvec; i += stride) __stcs(dst + i, v);
}

}  // namespace

cudaError_t kernels_init_device() {
  const int smem = (int)(kSmemFixed + 4 * kMaxSegsPerLaunch + 128);
  const cudaError_t e = cudaFuncSetAttribute(kk_convert_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(kk_convert_f16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
}

cudaError_t launch_convert(const ConvertLaunch& L, int sm_count, cudaStream_t stream) {
  if (L.n_tiles == 0) return cudaSuccess;
  if (L.n_segs == 0 || L.n_segs > kMaxSegsPerLaunch || L.n_dst == 0 || L.n_dst > KK_MAX_DST || !L.sched) return cudaErrorInvalidValue;
  const uint32_t grid = L.n_tiles < (uint32_t)sm_count ? L.n_tiles : (uint32_t)sm_count;
  const size_t smem = kSmemFixed + 4 * (size_t)L.n_segs + 16;
  if (L.flags & KK_LAUNCH_F16) kk_convert_f16_kernel<<<grid, kThreads, smem, stream>>>(L);
  else kk_convert_kernel<<<grid, kThreads, smem, stream>>>(L);
  return cudaGetLastError();
}

cudaError_t launch_checksum(const uint8_t* p, uint64_t nbytes, unsigned long long* out, int sm_count, cudaStream_t stream) {
  if (nbytes == 0) return cudaSuccess;
  uint64_t want = (nbytes / 8 + 255) / 256;
  uint32_t grid = (uint32_t)(want < (uint64_t)sm_count * 8 ? (want ? want : 1) : (uint64_t)sm_count * 8);
  kk_checksum_kernel<<<grid, 256, 0, stream>>>(p, nbytes, out);
  return cudaGetLastError();
}

cudaError_t launch_ldg_copy(const uint8_t* src, uint8_t* dst, uint64_t nbytes, int sm_count, cudaStream_t stream) {
  if (nbytes == 0) return cudaSuccess;
  if ((nbytes & 15) || ((uintptr_t)src & 15) || ((uintptr_t)dst & 15)) return cudaErrorInvalidValue;
  kk_ldg_copy_kernel<<<sm_count * 8, 256, 0, stream>>>(reinterpret_cast<const uint4*>(src), reinterpret_cast<uint4*>(dst), nbytes >> 4);
  return cudaGetLastError();
}

}  // namespace kk

namespace kk {
cudaError_t launch_fill(uint8_t* dst, uint64_t nbytes, int sm_count, cudaStream_t stream) {
  if (nbytes == 0) return cudaSuccess;
  if ((nbytes & 15) || ((uintptr_t)dst & 15)) return cudaErrorInvalidValue;
  kk_fill_kernel<<<sm_count * 8, 256, 0, stream>>>(reinterpret_cast<uint4*>(dst), nbytes >> 4, make_uint4(0x3F803F80u, 0x3F803F80u, 0x3F803F80u, 0x3F803F80u));
  return cudaGetLastError();
}
}  // namespace kk
