// Per-tile work description of kk_convert_kernel, as ONE function the device and the host both run: which bytes a tile pulls into its
// stage (one bulk copy of a 16-byte aligned superset, or one bulk copy per source row for the transposes) and the descriptor the consumer
// warps act on.  The kernel's producer warp calls it for every tile, and tests/emul replays whole launches through the same function
// (kk_emul_launch) — planner output in, pool bytes out, device source in between — so the CPU tier and the GPU run one transcription.
#pragma once
#include "kk_ops.h"

struct alignas(16) KKTileDesc {
  uint32_t op;
  uint32_t pay_off;  // payload offset inside the stage buffer (0..15 for TMA tiles)
  uint32_t n_units;  // units in this tile (bytes / elements / blocks); transposes: rows | cols<<16
  uint32_t bulk;     // 1: aligned copy, bulk-store from shared memory; 3: row-split exchange; 4: transpose tile staged by bulk copies, rows nc*es bytes apart
                     // (0 for a transpose tile = not staged: the consumers gather it themselves)
  uint64_t dst_off;  // pool byte offset of the tile's first output (transposes: dst tensor origin)
  uint64_t src_off;  // transposes: byte offset of source element (r0, c0) from the launch's src base
  uint32_t C;        // transposes: source columns
  uint32_t R;        // transposes: destination row length
  uint32_t col0;     // transposes: first source column of the tile
  uint32_t row0;     // transposes: first destination column (= global source row) of the tile
  uint32_t pad[4];
};
static_assert(sizeof(KKTileDesc) == 64, "KKTileDesc");

// What the producer issues for the tile.  kind 0: nothing (the consumers gather the tile themselves, or it is empty);
// kind 1: one bulk copy of `tx` bytes from src + g_off (16-byte aligned) to the start of the stage;
// kind 2: `nrows` bulk copies of `row_bytes` from src + g_off + r * gpitch to stage + r * spitch.  tx is always the total byte count.
// pay: the payload bytes among them, from the descriptor's pay_off on; the rest of a kind-1 copy (tx - pay_off - pay, at most 15 bytes) is the
// 16-byte rounding of the superset, which the consumers must not depend on.
struct KKTileLoad {
  uint32_t kind, tx;
  uint64_t g_off;
  uint32_t nrows, row_bytes, spitch, pay;
  uint64_t gpitch;
};

// seg: the segment tile `t` (counted from the segment's first tile) belongs to; src_addr: address of the launch's src base (only its
// alignment matters); flags: ConvertLaunch::flags.
static inline KK_HD void kk_make_tile(const KKSeg& seg, uint32_t t, uint64_t src_addr, uint32_t flags, KKTileDesc& d, KKTileLoad& ld) {
  d.op = seg.op; d.pay_off = 0; d.n_units = 0; d.bulk = 0; d.dst_off = 0; d.src_off = 0; d.C = 0; d.R = 0; d.col0 = 0; d.row0 = 0;
  ld.kind = 0; ld.tx = 0; ld.g_off = 0; ld.nrows = 0; ld.row_bytes = 0; ld.spitch = 0; ld.pay = 0; ld.gpitch = 0;
  uint32_t in_bytes = 0;  // source bytes of this tile (single-copy ops)
  uint64_t in_off = 0;    // their offset from the src base
  uint32_t t_es = 0;  // transposes: source element size
  switch (seg.op) {
    case KK_OP_COPY:
    case KK_OP_ROWSPLIT: {
      const uint64_t o = (uint64_t)t * KK_TILE_SRC_BYTES;
      const uint64_t rem = seg.units - o;
      d.n_units = rem < KK_TILE_SRC_BYTES ? (uint32_t)rem : KK_TILE_SRC_BYTES;
      in_bytes = d.n_units; in_off = seg.src_off + o;
      if (seg.op == KK_OP_COPY) {
        d.dst_off = seg.dst_off + o;
      } else {
        d.dst_off = seg.dst_off;
        d.C = seg.p0;                   // row bytes
        d.R = seg.p1;                   // slice bytes
        d.row0 = seg.p2;                // first row of this rank's piece
        d.col0 = seg.p3 + (uint32_t)o;  // byte position of the tile inside the piece
      }
      break;
    }
    case KK_OP_F8E4M3_BF16:
    case KK_OP_F8E5M2_BF16: {
      const uint64_t e = (uint64_t)t * KK_TILE_SRC_BYTES;
      const uint64_t rem = seg.units - e;
      d.n_units = rem < KK_TILE_SRC_BYTES ? (uint32_t)rem : KK_TILE_SRC_BYTES;
      in_bytes = d.n_units; in_off = seg.src_off + e; d.dst_off = seg.dst_off + e * 2;
      break;
    }
    case KK_OP_F32_BF16: {
      const uint64_t e = (uint64_t)t * (KK_TILE_SRC_BYTES / 4);
      const uint64_t rem = seg.units - e;
      d.n_units = rem < KK_TILE_SRC_BYTES / 4 ? (uint32_t)rem : KK_TILE_SRC_BYTES / 4;
      in_bytes = d.n_units * 4; in_off = seg.src_off + e * 4; d.dst_off = seg.dst_off + e * 2;
      break;
    }
    case KK_OP_F16_BF16: {
      const uint64_t e = (uint64_t)t * (KK_TILE_SRC_BYTES / 2);
      const uint64_t rem = seg.units - e;
      d.n_units = rem < KK_TILE_SRC_BYTES / 2 ? (uint32_t)rem : KK_TILE_SRC_BYTES / 2;
      in_bytes = d.n_units * 2; in_off = seg.src_off + e * 2; d.dst_off = seg.dst_off + e * 2;
      break;
    }
    case KK_OP_T_F32_BF16: case KK_OP_T_B32: case KK_OP_T_F16_BF16: case KK_OP_T_B16: t_es = kk_t_src_es(seg.op); break;
    default: {  // block-dequantising ops
      const KKBlockGeom g = kk_block_geom(seg.op);
      if (g.block_bytes) {
        const KKBlockTile bt = kk_block_tile(seg, t);
        d.n_units = bt.n_blocks;
        in_bytes = bt.in_bytes; in_off = bt.in_off;
        d.dst_off = bt.dst_off;
      }
      break;
    }
  }
  if (t_es) {  // rows x columns window of the source matrix, staged row by row when every row piece is a whole number of aligned 16-byte units
    const uint32_t C = seg.p0, W = kk_t_width(seg.op, C);
    const uint32_t ct = (C + W - 1) / W;
    const uint32_t tr = t / ct, tc = t % ct;
    const uint64_t r0 = (uint64_t)tr * KK_T_ROWS;
    const uint32_t c0 = tc * W;
    const uint64_t rrem = seg.units - r0;
    const uint32_t nr = rrem < KK_T_ROWS ? (uint32_t)rrem : KK_T_ROWS;
    const uint32_t nc = (C - c0) < W ? (C - c0) : W;
    d.n_units = nr | (nc << 16);
    d.C = C; d.R = seg.p1; d.col0 = c0; d.row0 = seg.p2 + (uint32_t)r0;
    d.src_off = seg.src_off + (r0 * C + c0) * t_es;
    d.dst_off = seg.dst_off;
    const uint64_t row_pitch = (uint64_t)C * t_es;
    const uint32_t rb = nc * t_es;
    if (((src_addr + d.src_off) & 15u) == 0 && (row_pitch & 15u) == 0 && (rb & 15u) == 0) {
      d.bulk = 4;
      ld.tx = ld.pay = nr * rb;
      ld.g_off = d.src_off;
      if (nc == C) {  // the tile spans whole rows: they are contiguous in the source, one bulk copy brings all of them
        ld.kind = 1;
      } else {
        ld.kind = 2;
        ld.nrows = nr; ld.row_bytes = rb; ld.spitch = rb; ld.gpitch = row_pitch;
      }
    }
    return;  // not staged: descriptor only, the consumers gather the tile themselves
  }
  if (in_bytes) {
    const uint32_t mis = (uint32_t)((src_addr + in_off) & 15u);
    d.pay_off = mis;
    ld.kind = 1;
    ld.tx = (mis + in_bytes + 15u) & ~15u;
    ld.pay = in_bytes;
    ld.g_off = in_off - mis;
    if (seg.op == KK_OP_COPY && mis == 0 && (in_bytes & 15u) == 0 && !(flags & KK_LAUNCH_MULTIMEM)) d.bulk = 1;
    // row-split exchange: every (row, destination) piece must be a whole number of 16-byte units on both sides
    if (seg.op == KK_OP_ROWSPLIT && mis == 0 && (seg.p0 & 15u) == 0 && (seg.p1 & 15u) == 0 && (in_bytes & 15u) == 0 && (seg.dst_off & 15u) == 0)
      d.bulk = 3;
  }
}

// The segment tile `tile` belongs to: the last one whose tile_begin is <= tile, searched forward from `cur` (a CTA's tiles only increase).
static inline KK_HD uint32_t kk_tile_seg(const uint32_t* tile_begin, uint32_t n_segs, uint32_t cur, uint32_t tile) {
  while (cur + 1 < n_segs && tile_begin[cur + 1] <= tile) ++cur;
  return cur;
}

// Row-split exchange (KK_OP_ROWSPLIT) addressing, shared by the kernel's two consumers and tests/emul.  A tile holds n_units bytes of this
// rank's piece from byte col0 of it on; the piece is whole source rows of C bytes, tensor row row0 first.  Column `col` of piece row `row`
// belongs to rank j = col / R and lands in that rank's pool at dst_off + (row0 + row) * R + col % R.
struct KKRowSplitDst {
  uint32_t j;       // destination rank (index into ConvertLaunch::xdst)
  uint32_t within;  // column inside the rank's slice
  uint64_t off;     // byte offset in that rank's pool
};
static inline KK_HD KKRowSplitDst kk_rowsplit_col(const KKTileDesc& d, uint32_t col) {  // rank and column in its slice; off is left 0
  KKRowSplitDst x;
  x.j = col / d.R;
  x.within = col - x.j * d.R;
  x.off = 0;
  return x;
}
static inline KK_HD uint64_t kk_rowsplit_off(const KKTileDesc& d, uint32_t row, uint32_t within) {
  return d.dst_off + (uint64_t)(d.row0 + row) * d.R + within;
}

// Byte k of the tile (the byte-granular consumer).
static inline KK_HD KKRowSplitDst kk_rowsplit_byte(const KKTileDesc& d, uint32_t k) {
  const uint32_t pos = d.col0 + k;
  const uint32_t row = pos / d.C;
  KKRowSplitDst x = kk_rowsplit_col(d, pos - row * d.C);
  x.off = kk_rowsplit_off(d, row, x.within);
  return x;
}

// The (row, destination rank) pieces of a tile, in order (the bulk-store consumer, t.bulk == 3): each piece is the longest run of the tile's
// bytes inside one row and one slice.
//   for (KKRowSplitWalk w = kk_rowsplit_walk(d); w.pos < w.end;) { p = kk_rowsplit_piece(d, w); <store p>; kk_rowsplit_advance(d, w, p.len); }
struct KKRowSplitWalk {
  uint32_t pos, end, row, col;  // byte position of the next piece in this rank's piece, end of the tile, the next piece's row and column
};
struct KKRowSplitPiece {
  KKRowSplitDst dst;
  uint32_t len;
  uint32_t src;  // offset of the piece's first byte from the tile's payload
};
static inline KK_HD KKRowSplitWalk kk_rowsplit_walk(const KKTileDesc& d) {
  KKRowSplitWalk w;
  w.pos = d.col0;
  w.end = d.col0 + d.n_units;
  w.row = w.pos / d.C;
  w.col = w.pos - w.row * d.C;
  return w;
}
static inline KK_HD KKRowSplitPiece kk_rowsplit_piece(const KKTileDesc& d, const KKRowSplitWalk& w) {
  KKRowSplitPiece p;
  p.dst = kk_rowsplit_col(d, w.col);
  p.len = d.R - p.dst.within;
  if (p.len > w.end - w.pos) p.len = w.end - w.pos;
  p.dst.off = kk_rowsplit_off(d, w.row, p.dst.within);
  p.src = w.pos - d.col0;
  return p;
}
static inline KK_HD void kk_rowsplit_advance(const KKTileDesc& d, KKRowSplitWalk& w, uint32_t len) {
  w.pos += len;
  w.col += len;
  const bool wrap = w.col >= d.C;
  w.row += wrap;
  w.col = wrap ? 0u : w.col;
}
