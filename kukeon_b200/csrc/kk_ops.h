// Shared between the host planner and the device kernels: the per-launch segment table and the
// tile geometry.  A *segment* is one contiguous run of one tensor inside one staged chunk; a *tile*
// is the unit a CTA pulls through shared memory (<= KK_TILE_SRC_BYTES of source).
#pragma once
#include <stdint.h>

#define KK_TILE_SRC_BYTES 32768u /* payload bytes per smem stage */
#define KK_STAGE_PAD 128u        /* slack so a 16-B-aligned superset of a misaligned tile still fits */
#define KK_Q4K_BLOCK_BYTES 144u
#define KK_Q4K_BLOCK_ELEMS 256u
#define KK_Q4K_TILE_BLOCKS 224u  /* 224*144 = 32256 B in, 224*512 = 114688 B out.  16 consumer warps x 4 blocks = 64 blocks per sweep, so 3.5 sweeps; timed
                                    against 192-block tiles (3 full sweeps), contiguous 14-block runs per warp, a rotated warp order, 20 warps and, under
                                    dynamic tile scheduling, 186-223 blocks: none faster, so the simplest form stays */
#define KK_Q8_0_BLOCK_BYTES 34u
#define KK_Q8_0_BLOCK_ELEMS 32u
#define KK_Q8_0_TILE_BLOCKS 960u /* 960*34 = 32640 B in (a multiple of 16), 960*64 = 61440 B out */
#define KK_Q6K_BLOCK_BYTES 210u
#define KK_Q6K_TILE_BLOCKS 152u  /* 152*210 = 31920 B in (a multiple of 16), 152*512 = 77824 B out */
/* §8(f4) legacy and K quants: blocks per tile chosen so that a full tile's source bytes are a multiple of 16 (every tile
 * of a 16-byte aligned tensor then starts 16-byte aligned in its stage) and at most KK_TILE_SRC_BYTES. */
#define KK_Q4_0_BLOCK_BYTES 18u
#define KK_Q4_0_TILE_BLOCKS 1816u /* 32688 B in, 116224 B out */
#define KK_Q4_1_BLOCK_BYTES 20u
#define KK_Q4_1_TILE_BLOCKS 1632u /* 32640 B in */
#define KK_Q5_0_BLOCK_BYTES 22u
#define KK_Q5_0_TILE_BLOCKS 1488u /* 32736 B in */
#define KK_Q5_1_BLOCK_BYTES 24u
#define KK_Q5_1_TILE_BLOCKS 1360u /* 32640 B in */
#define KK_Q2K_BLOCK_BYTES 84u
#define KK_Q2K_TILE_BLOCKS 388u   /* 32592 B in, 198656 B out */
#define KK_Q3K_BLOCK_BYTES 110u
#define KK_Q3K_TILE_BLOCKS 296u   /* 32560 B in */
#define KK_Q5K_BLOCK_BYTES 176u
#define KK_Q5K_TILE_BLOCKS 186u   /* 32736 B in */
#define KK_IQ4NL_BLOCK_BYTES 18u
#define KK_IQ4NL_TILE_BLOCKS 1816u /* as Q4_0 */
#define KK_IQ4XS_BLOCK_BYTES 136u
#define KK_IQ4XS_TILE_BLOCKS 240u  /* 32640 B in */
#define KK_MXFP4_BLOCK_BYTES 17u
#define KK_MXFP4_TILE_BLOCKS 1920u /* 32640 B in */
/* lattice i-quants, ternary types, NVFP4: blocks per tile chosen like the others (full tile <= KK_TILE_SRC_BYTES, a multiple of 16 bytes) */
#define KK_IQ2XXS_BLOCK_BYTES 66u
#define KK_IQ2XXS_TILE_BLOCKS 496u /* 32736 B in */
#define KK_IQ2XS_BLOCK_BYTES 74u
#define KK_IQ2XS_TILE_BLOCKS 440u /* 32560 B in */
#define KK_IQ2S_BLOCK_BYTES 82u
#define KK_IQ2S_TILE_BLOCKS 392u /* 32144 B in */
#define KK_IQ3XXS_BLOCK_BYTES 98u
#define KK_IQ3XXS_TILE_BLOCKS 328u /* 32144 B in */
#define KK_IQ3S_BLOCK_BYTES 110u
#define KK_IQ3S_TILE_BLOCKS 296u /* 32560 B in */
#define KK_IQ1S_BLOCK_BYTES 50u
#define KK_IQ1S_TILE_BLOCKS 648u /* 32400 B in */
#define KK_IQ1M_BLOCK_BYTES 56u
#define KK_IQ1M_TILE_BLOCKS 584u /* 32704 B in */
#define KK_TQ1_0_BLOCK_BYTES 54u
#define KK_TQ1_0_TILE_BLOCKS 600u /* 32400 B in */
#define KK_TQ2_0_BLOCK_BYTES 66u
#define KK_TQ2_0_TILE_BLOCKS 496u /* 32736 B in */
#define KK_NVFP4_BLOCK_BYTES 36u
#define KK_NVFP4_TILE_BLOCKS 908u /* 32688 B in */
/* 2-D transposes (GPT-2 Conv1D): a tile is 8 source rows x up to KK_T_ROW_BYTES of each.  Eight bulk copies bring in a full 32 KiB stage (ONE when the
 * tile spans whole rows, which are then contiguous in the source); consumers read along rows — conflict-free at any pitch — and every thread packs
 * the 8 rows of one column into a single 16-byte store.  Timed on GPT-2-small against 32x128 tiles and 32-row x 960-byte wide-store tiles, both
 * slower — the other two geometries are gone. */
#define KK_T_ROWS 8u             /* a multiple of 8; 16 x 2 KiB and 32 x 1 KiB tiles (whole-sector stores per thread) are slower on GPT-2-small */
#define KK_T_ROW_BYTES 4096u     /* per staged row: 1024 32-bit or 2048 16-bit columns */
#define KK_MAX_DST 8
/* ConvertLaunch::flags */
#define KK_LAUNCH_NO_BULK_STORE 0x1u  /* force the register path for aligned copies (A/B measurement) */
#define KK_LAUNCH_MULTIMEM 0x2u       /* dst[0] is an NVLS multicast address: store with multimem.st */

enum KKOp : uint32_t {
  KK_OP_COPY = 0,      // units = bytes
  KK_OP_F32_BF16 = 1,  // units = elements
  KK_OP_F16_BF16 = 2,  // units = elements
  KK_OP_Q4K_BF16 = 3,  // units = 256-weight blocks
  // 2-D transposes on 8-row tiles: units = source rows in this segment, p0 = source columns (elements),
  // p1 = destination row length in elements (= total source rows of the tensor),
  // p2 = index of this segment's first source row (destination column offset).
  KK_OP_T_F32_BF16 = 4,
  KK_OP_T_F16_BF16 = 5,
  KK_OP_T_B16 = 6,     // 2-byte elements moved verbatim (bf16, i16, ...)
  KK_OP_T_B32 = 7,     // 4-byte elements moved verbatim (F32 under KK_LOAD_KEEP_F32, i32, ...)
  KK_OP_Q8_0_BF16 = 8, // units = 32-weight blocks (34 B: d f16 | 32 x int8)
  KK_OP_Q6K_BF16 = 9,  // units = 256-weight super-blocks (210 B: ql[128] | qh[64] | scales[16] int8 | d f16)
  // SCATTER exchange: units = bytes of whole source rows; every row is cut into N column slices of p1 bytes and slice j
  // goes to pool j (ConvertLaunch::xdst[j]) at dst_off + row * p1.  p0 = row bytes, p1 = slice bytes, p2 = index of the
  // first row of this rank's piece, p3 = bytes of the piece that precede this segment.
  KK_OP_ROWSPLIT = 10,
  // units = 32-weight blocks: Q4_0 (18 B: d f16 | qs[16]), Q4_1 (20 B: d | m | qs), Q5_0 (22 B: d | qh u32 | qs), Q5_1 (24 B: d | m | qh | qs)
  KK_OP_Q4_0_BF16 = 11,
  KK_OP_Q4_1_BF16 = 12,
  KK_OP_Q5_0_BF16 = 13,
  KK_OP_Q5_1_BF16 = 14,
  // units = 256-weight super-blocks: Q2_K (84 B: scales[16] | qs[64] | d | dmin), Q3_K (110 B: hmask[32] | qs[64] | scales[12] | d),
  // Q5_K (176 B: d | dmin | scales[12] | qh[32] | qs[128])
  KK_OP_Q2K_BF16 = 15,
  KK_OP_Q3K_BF16 = 16,
  KK_OP_Q5K_BF16 = 17,
  // units = elements (1 byte each): FP8 widened to bf16 (KK_LOAD_F8_TO_BF16)
  KK_OP_F8E4M3_BF16 = 18,
  KK_OP_F8E5M2_BF16 = 19,
  // 20..22 and 26..28 were the two candidate transpose geometries of round 1 (retired after the round-2 A/B; numbers not reused)
  // codebook 4-bit types: IQ4_NL (18 B: d f16 | qs[16]), IQ4_XS (136 B: d | scales_h u16 | scales_l[4] | qs[128]), MXFP4 (17 B: E8M0 | qs[16])
  KK_OP_IQ4NL_BF16 = 23,
  KK_OP_IQ4XS_BF16 = 24,
  KK_OP_MXFP4_BF16 = 25,
  // lattice i-quants (256-weight super-blocks; 8 weights = one grid entry of kk_iq_grids.h, or two 4-value entries for IQ3), the ternary
  // types, and NVFP4 (64-weight blocks: 4 UE4M3 scales | 32 nibble bytes)
  KK_OP_IQ2XXS_BF16 = 29,
  KK_OP_IQ2XS_BF16 = 30,
  KK_OP_IQ2S_BF16 = 31,
  KK_OP_IQ3XXS_BF16 = 32,
  KK_OP_IQ3S_BF16 = 33,
  KK_OP_IQ1S_BF16 = 34,
  KK_OP_IQ1M_BF16 = 35,
  KK_OP_TQ1_0_BF16 = 36,
  KK_OP_TQ2_0_BF16 = 37,
  KK_OP_NVFP4_BF16 = 38,
  KK_OP_COUNT = 39,
  KK_OP_END = 0xFFFFFFFFu  // never in a segment table: the producer warp's end-of-work marker in the stage descriptor ring
};

struct KKSeg {
  uint64_t src_off;    // byte offset of the segment's first source byte from the launch's src base
  uint64_t dst_off;    // byte offset into the pool (for transposes: of the destination tensor's origin)
  uint64_t units;      // op-specific, see KKOp
  uint32_t op;
  uint32_t tile_begin; // index of this segment's first tile within the launch
  uint32_t p0, p1, p2, p3;
};

#ifdef __cplusplus
static_assert(sizeof(KKSeg) == 48, "KKSeg layout is shared with the device");

#ifdef __CUDACC__
#define KK_HD __host__ __device__
#else
#define KK_HD
#endif

// Geometry of the block-dequantising ops: source bytes and bf16 output bytes per block, blocks per tile.
// block_bytes == 0: `op` is not a block op.
struct KKBlockGeom {
  uint32_t block_bytes, out_bytes, tile_blocks;
};
static inline KK_HD bool kk_is_transpose(uint32_t op) { return op >= KK_OP_T_F32_BF16 && op <= KK_OP_T_B32; }
static inline KK_HD uint32_t kk_t_src_es(uint32_t op) { return (op == KK_OP_T_F32_BF16 || op == KK_OP_T_B32) ? 4u : 2u; }
/* Columns per 8-row tile of a tensor with C source columns: at most what a staged row holds (1024 32-bit / 2048 16-bit), and rows wider than that
 * are cut into EQUAL pieces (2304 columns -> 768 + 768 + 768, not 1024 + 1024 + 256: with a fixed width every third tile of GPT-2's c_attn would be a
 * quarter full and still cost a pipeline slot), rounded up to 8 columns so that row pieces stay whole 16-byte units for either element size. */
static inline KK_HD uint32_t kk_t_width(uint32_t op, uint32_t C) {
  const uint32_t wmax = KK_T_ROW_BYTES / kk_t_src_es(op);
  if (C > wmax) {
    const uint32_t n = (C + wmax - 1u) / wmax;
    const uint32_t w = ((C + n - 1u) / n + 7u) & ~7u;
    return w < wmax ? w : wmax;
  }
  return wmax;
}

static inline KK_HD KKBlockGeom kk_block_geom(uint32_t op) {
  switch (op) {
    case KK_OP_Q4K_BF16: return {KK_Q4K_BLOCK_BYTES, 512u, KK_Q4K_TILE_BLOCKS};
    case KK_OP_Q8_0_BF16: return {KK_Q8_0_BLOCK_BYTES, 64u, KK_Q8_0_TILE_BLOCKS};
    case KK_OP_Q6K_BF16: return {KK_Q6K_BLOCK_BYTES, 512u, KK_Q6K_TILE_BLOCKS};
    case KK_OP_Q4_0_BF16: return {KK_Q4_0_BLOCK_BYTES, 64u, KK_Q4_0_TILE_BLOCKS};
    case KK_OP_Q4_1_BF16: return {KK_Q4_1_BLOCK_BYTES, 64u, KK_Q4_1_TILE_BLOCKS};
    case KK_OP_Q5_0_BF16: return {KK_Q5_0_BLOCK_BYTES, 64u, KK_Q5_0_TILE_BLOCKS};
    case KK_OP_Q5_1_BF16: return {KK_Q5_1_BLOCK_BYTES, 64u, KK_Q5_1_TILE_BLOCKS};
    case KK_OP_Q2K_BF16: return {KK_Q2K_BLOCK_BYTES, 512u, KK_Q2K_TILE_BLOCKS};
    case KK_OP_Q3K_BF16: return {KK_Q3K_BLOCK_BYTES, 512u, KK_Q3K_TILE_BLOCKS};
    case KK_OP_Q5K_BF16: return {KK_Q5K_BLOCK_BYTES, 512u, KK_Q5K_TILE_BLOCKS};
    case KK_OP_IQ4NL_BF16: return {KK_IQ4NL_BLOCK_BYTES, 64u, KK_IQ4NL_TILE_BLOCKS};
    case KK_OP_IQ4XS_BF16: return {KK_IQ4XS_BLOCK_BYTES, 512u, KK_IQ4XS_TILE_BLOCKS};
    case KK_OP_MXFP4_BF16: return {KK_MXFP4_BLOCK_BYTES, 64u, KK_MXFP4_TILE_BLOCKS};
    case KK_OP_IQ2XXS_BF16: return {KK_IQ2XXS_BLOCK_BYTES, 512u, KK_IQ2XXS_TILE_BLOCKS};
    case KK_OP_IQ2XS_BF16: return {KK_IQ2XS_BLOCK_BYTES, 512u, KK_IQ2XS_TILE_BLOCKS};
    case KK_OP_IQ2S_BF16: return {KK_IQ2S_BLOCK_BYTES, 512u, KK_IQ2S_TILE_BLOCKS};
    case KK_OP_IQ3XXS_BF16: return {KK_IQ3XXS_BLOCK_BYTES, 512u, KK_IQ3XXS_TILE_BLOCKS};
    case KK_OP_IQ3S_BF16: return {KK_IQ3S_BLOCK_BYTES, 512u, KK_IQ3S_TILE_BLOCKS};
    case KK_OP_IQ1S_BF16: return {KK_IQ1S_BLOCK_BYTES, 512u, KK_IQ1S_TILE_BLOCKS};
    case KK_OP_IQ1M_BF16: return {KK_IQ1M_BLOCK_BYTES, 512u, KK_IQ1M_TILE_BLOCKS};
    case KK_OP_TQ1_0_BF16: return {KK_TQ1_0_BLOCK_BYTES, 512u, KK_TQ1_0_TILE_BLOCKS};
    case KK_OP_TQ2_0_BF16: return {KK_TQ2_0_BLOCK_BYTES, 512u, KK_TQ2_0_TILE_BLOCKS};
    case KK_OP_NVFP4_BF16: return {KK_NVFP4_BLOCK_BYTES, 128u, KK_NVFP4_TILE_BLOCKS};
    default: return {0u, 0u, 0u};
  }
}
// Tile t of a block-op segment: the blocks it covers, where their bytes start (relative to the launch's src base) and
// where their bf16 output starts in the pool.  Used by the kernel's producer warp and by tests/emul.
struct KKBlockTile {
  uint32_t n_blocks, in_bytes;
  uint64_t in_off, dst_off;
};
static inline KK_HD KKBlockTile kk_block_tile(const KKSeg& seg, uint32_t t) {
  const KKBlockGeom g = kk_block_geom(seg.op);
  const uint64_t b = (uint64_t)t * g.tile_blocks;
  const uint64_t rem = seg.units - b;
  KKBlockTile r;
  r.n_blocks = rem < g.tile_blocks ? (uint32_t)rem : g.tile_blocks;
  r.in_bytes = r.n_blocks * g.block_bytes;
  r.in_off = seg.src_off + b * g.block_bytes;
  r.dst_off = seg.dst_off + b * g.out_bytes;
  return r;
}
#define KK_TILE_OK(bytes, blocks) ((bytes) * (blocks) <= KK_TILE_SRC_BYTES && ((bytes) * (blocks)) % 16u == 0)
static_assert(KK_TILE_OK(KK_Q4K_BLOCK_BYTES, KK_Q4K_TILE_BLOCKS) && KK_TILE_OK(KK_Q8_0_BLOCK_BYTES, KK_Q8_0_TILE_BLOCKS) &&
                  KK_TILE_OK(KK_Q6K_BLOCK_BYTES, KK_Q6K_TILE_BLOCKS) && KK_TILE_OK(KK_Q4_0_BLOCK_BYTES, KK_Q4_0_TILE_BLOCKS) &&
                  KK_TILE_OK(KK_Q4_1_BLOCK_BYTES, KK_Q4_1_TILE_BLOCKS) && KK_TILE_OK(KK_Q5_0_BLOCK_BYTES, KK_Q5_0_TILE_BLOCKS) &&
                  KK_TILE_OK(KK_Q5_1_BLOCK_BYTES, KK_Q5_1_TILE_BLOCKS) && KK_TILE_OK(KK_Q2K_BLOCK_BYTES, KK_Q2K_TILE_BLOCKS) &&
                  KK_TILE_OK(KK_Q3K_BLOCK_BYTES, KK_Q3K_TILE_BLOCKS) && KK_TILE_OK(KK_Q5K_BLOCK_BYTES, KK_Q5K_TILE_BLOCKS) &&
                  KK_TILE_OK(KK_IQ4NL_BLOCK_BYTES, KK_IQ4NL_TILE_BLOCKS) && KK_TILE_OK(KK_IQ4XS_BLOCK_BYTES, KK_IQ4XS_TILE_BLOCKS) &&
                  KK_TILE_OK(KK_MXFP4_BLOCK_BYTES, KK_MXFP4_TILE_BLOCKS) &&
                  KK_TILE_OK(KK_IQ2XXS_BLOCK_BYTES, KK_IQ2XXS_TILE_BLOCKS) && KK_TILE_OK(KK_IQ2XS_BLOCK_BYTES, KK_IQ2XS_TILE_BLOCKS) &&
                  KK_TILE_OK(KK_IQ2S_BLOCK_BYTES, KK_IQ2S_TILE_BLOCKS) && KK_TILE_OK(KK_IQ3XXS_BLOCK_BYTES, KK_IQ3XXS_TILE_BLOCKS) &&
                  KK_TILE_OK(KK_IQ3S_BLOCK_BYTES, KK_IQ3S_TILE_BLOCKS) && KK_TILE_OK(KK_IQ1S_BLOCK_BYTES, KK_IQ1S_TILE_BLOCKS) &&
                  KK_TILE_OK(KK_IQ1M_BLOCK_BYTES, KK_IQ1M_TILE_BLOCKS) && KK_TILE_OK(KK_TQ1_0_BLOCK_BYTES, KK_TQ1_0_TILE_BLOCKS) &&
                  KK_TILE_OK(KK_TQ2_0_BLOCK_BYTES, KK_TQ2_0_TILE_BLOCKS) && KK_TILE_OK(KK_NVFP4_BLOCK_BYTES, KK_NVFP4_TILE_BLOCKS),
              "a full tile of every block op fits one stage and keeps the next tile 16-byte aligned");

// Units one tile covers, and the number of tiles of a segment (host + device).
static inline KK_HD uint64_t kk_seg_tiles(uint32_t op, uint64_t units, uint32_t p0) {
  switch (op) {
    case KK_OP_COPY:
    case KK_OP_F8E4M3_BF16:
    case KK_OP_F8E5M2_BF16:
    case KK_OP_ROWSPLIT: return (units + KK_TILE_SRC_BYTES - 1) / KK_TILE_SRC_BYTES;
    case KK_OP_F32_BF16: return (units + KK_TILE_SRC_BYTES / 4 - 1) / (KK_TILE_SRC_BYTES / 4);
    case KK_OP_F16_BF16: return (units + KK_TILE_SRC_BYTES / 2 - 1) / (KK_TILE_SRC_BYTES / 2);
    case KK_OP_Q4K_BF16: return (units + KK_Q4K_TILE_BLOCKS - 1) / KK_Q4K_TILE_BLOCKS;
    case KK_OP_Q8_0_BF16: return (units + KK_Q8_0_TILE_BLOCKS - 1) / KK_Q8_0_TILE_BLOCKS;
    case KK_OP_Q6K_BF16: return (units + KK_Q6K_TILE_BLOCKS - 1) / KK_Q6K_TILE_BLOCKS;
    case KK_OP_Q4_0_BF16:
    case KK_OP_Q4_1_BF16:
    case KK_OP_Q5_0_BF16:
    case KK_OP_Q5_1_BF16:
    case KK_OP_Q2K_BF16:
    case KK_OP_Q3K_BF16:
    case KK_OP_Q5K_BF16:
    case KK_OP_IQ4NL_BF16:
    case KK_OP_IQ4XS_BF16:
    case KK_OP_IQ2XXS_BF16:
    case KK_OP_IQ2XS_BF16:
    case KK_OP_IQ2S_BF16:
    case KK_OP_IQ3XXS_BF16:
    case KK_OP_IQ3S_BF16:
    case KK_OP_IQ1S_BF16:
    case KK_OP_IQ1M_BF16:
    case KK_OP_TQ1_0_BF16:
    case KK_OP_TQ2_0_BF16:
    case KK_OP_NVFP4_BF16:
    case KK_OP_MXFP4_BF16: {
      const uint32_t tb = kk_block_geom(op).tile_blocks;
      return (units + tb - 1) / tb;
    }
    case KK_OP_T_F32_BF16:
    case KK_OP_T_B32:
    case KK_OP_T_F16_BF16:
    case KK_OP_T_B16: {
      const uint64_t w = kk_t_width(op, p0);
      return ((units + KK_T_ROWS - 1) / KK_T_ROWS) * (((uint64_t)p0 + w - 1) / w);
    }
    default: return 0;
  }
}
static_assert(KK_T_ROWS * KK_T_ROW_BYTES <= KK_TILE_SRC_BYTES, "a transpose tile fits a stage");
#endif
