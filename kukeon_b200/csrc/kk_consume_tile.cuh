// The per-tile walk of a kk_convert_kernel launch, as functions the device and the host both compile: the copies the producer issues for
// a tile (kk_load_tile), the bulk stores of the aligned copy and row-split tiles (kk_store_tile), and the consumer dispatch of every other
// tile — which per-lane body it runs and with which arguments (kk_consume_tile).  tests/emul plays whole launches through them, so the
// CPU tier checks this walk — the copies, the bulk-store pieces, the warp rotation, every op's template arguments, the transposes' gather
// and the row-split byte fallback — and not a copy of it.  What only the hardware needs (mbarriers, proxy fences, bulk-group commits and
// waits) stays in kk_kernels.cu.  Primitives: those of kk_dequant.cuh, and bulk_load / store_bulk / rowsplit_store_bulk below.
#pragma once
#include "kk_dequant.cuh"
#include "kk_tile.h"

// The producer's copies of tile load ld into stage S: one bulk copy (kind 1) or one per source row (kind 2), each through
// bulk_load(S, stage offset, source offset from the launch's src base, bytes).  Arming the stage's mbarrier with ld.tx is the caller's.
template <class Stage>
KK_DQ_DEV void kk_load_tile(const KKTileLoad& ld, const Stage& S) {
  if (ld.kind == 1) bulk_load(S, 0u, ld.g_off, ld.tx);
  else if (ld.kind == 2)
    for (uint32_t r = 0; r < ld.nrows; ++r) bulk_load(S, r * ld.spitch, ld.g_off + (uint64_t)r * ld.gpitch, ld.row_bytes);
}

// The bulk stores of a tile with t.bulk == 1 (aligned copy: the payload at pay to every destination pool, store_bulk(D, pool, offset,
// stage address, bytes)) or t.bulk == 3 (aligned row-split exchange: one store per (row, rank) piece, rowsplit_store_bulk(L, rank, offset,
// stage address, bytes)).  One lane issues them.  The destinations' type is a template parameter too, so that store_bulk and Dst::n are
// looked up only where the function is used: an includer that plays consumer tiles alone need not bind them.
template <class Dst, class Launch>
KK_DQ_DEV void kk_store_tile(const Dst& D, const KKTileDesc& t, uint32_t pay, const Launch& L) {
  if (t.bulk == 1) {
#pragma unroll
    for (int dd = 0; dd < KK_MAX_DST; ++dd)
      if (dd < (int)D.n) store_bulk(D, dd, t.dst_off, pay, t.n_units);
    return;
  }
  for (KKRowSplitWalk w = kk_rowsplit_walk(t); w.pos < w.end;) {
    const KKRowSplitPiece p = kk_rowsplit_piece(t, w);
    rowsplit_store_bulk(L, p.dst.j, p.dst.off, pay + p.src, p.len);
    kk_rowsplit_advance(t, w, p.len);
  }
}

// 2-D transpose tile (KK_OP_T_*): staged by the producer (t.bulk == 4) or, when a source row is not 16-byte aligned, gathered here.
template <bool F16, int ES, int CONV>
KK_DQ_DEV void run_t(const Dsts& D, const uint8_t* src, const KKTileDesc& t, uint32_t sbase, int ctid) {
  const uint32_t nr = t.n_units & 0xFFFFu, nc = t.n_units >> 16;
  uint32_t pitch = nc * ES;
  if (t.bulk != 4) {
    pitch = (pitch + 3u) & ~3u;
    t_gather<ES>(src + t.src_off, sbase, pitch, nr, nc, t.C, ctid);
    named_bar_consumers();
  }
  consume_t<F16, ES, CONV>(D, sbase, pitch, nr, nc, t.R, t.col0, t.row0, t.dst_off, ctid);
}

// One tile t, staged at sbase with its payload at pay, for consumer thread ctid = 32 * cwarp + lane.  L is the launch (the kernel's
// ConvertLaunch): transposes gather from L.src, and row-split bytes go to rowsplit_store1(L, ...).  it counts the tiles this CTA's consumers
// have taken, and selects the warp rotation.  F16: the launch's output format (KK_LAUNCH_F16), which every converting body is instantiated
// for; the op codes name the default, bf16 output, which is also the default instantiation.
template <bool F16 = false, class Launch>
KK_DQ_DEV void kk_consume_tile(const Dsts& D, const KKTileDesc& t, uint32_t sbase, uint32_t pay, const Launch& L, int cwarp, int lane, int ctid,
                               uint32_t it) {
  // Block ops deal a tile's blocks (or groups of 4 / 8) to the 16 warps round-robin, and a full tile is rarely a multiple of 16 groups: a Q4_K tile
  // is 56 quads — warps 0-7 would take 4 on EVERY tile, warps 8-15 three, and the pipeline runs at the pace of the busier half (0.875: exactly
  // where Q4_K sat while Q5_K, whose 46.5 quads split almost evenly, reached 0.96 on the same code).  Rotating the warp numbering by half the
  // warps on odd tiles gives every warp 4 + 3 over two tiles; outputs depend on the block, not on which warp expands it.
  const int rwarp = (cwarp + (int)(it & 1u) * (kConsumerWarps / 2)) % kConsumerWarps;
  switch (t.op) {
    case KK_OP_ROWSPLIT: {  // unaligned fallback: byte-granular all-to-all copy
      for (uint32_t k = ctid; k < t.n_units; k += kConsumerThreads) {
        const KKRowSplitDst x = kk_rowsplit_byte(t, k);
        rowsplit_store1(L, x.j, x.off, (uint8_t)lds8(pay + k));
      }
      break;
    }
    case KK_OP_COPY: consume_copy(D, pay, t.n_units, t.dst_off, ctid); break;
    case KK_OP_F32_BF16: consume_f32<F16>(D, pay, t.n_units, t.dst_off, ctid); break;
    case KK_OP_F16_BF16: consume_f16<F16>(D, pay, t.n_units, t.dst_off, ctid); break;
    case KK_OP_Q4K_BF16: consume_q4k<F16>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_Q8_0_BF16: consume_q8_0<F16>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_Q6K_BF16: consume_q6k<F16>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_Q4_0_BF16: consume_legacy32<F16, KK_Q4_0_BLOCK_BYTES, false, false>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_Q4_1_BF16: consume_legacy32<F16, KK_Q4_1_BLOCK_BYTES, true, false>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_Q5_0_BF16: consume_legacy32<F16, KK_Q5_0_BLOCK_BYTES, false, true>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_Q5_1_BF16: consume_legacy32<F16, KK_Q5_1_BLOCK_BYTES, true, true>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_Q2K_BF16: consume_q2k<F16>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_Q3K_BF16: consume_q3k<F16>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_Q5K_BF16: consume_q5k<F16>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_IQ4NL_BF16: consume_codebook32<F16, KK_IQ4NL_BLOCK_BYTES, 0>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_MXFP4_BF16: consume_codebook32<F16, KK_MXFP4_BLOCK_BYTES, 1>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_IQ4XS_BF16: consume_iq4xs<F16>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_IQ2XXS_BF16: consume_iq2xxs<F16>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_IQ2XS_BF16: consume_iq2xs<F16>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_IQ2S_BF16: consume_iq2s<F16>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_IQ3XXS_BF16: consume_iq3xxs<F16>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_IQ3S_BF16: consume_iq3s<F16>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_IQ1S_BF16: consume_iq1s<F16>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_IQ1M_BF16: consume_iq1m<F16>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_TQ1_0_BF16: consume_tq1_0<F16>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_TQ2_0_BF16: consume_tq2_0<F16>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_NVFP4_BF16: consume_nvfp4<F16>(D, pay, t.n_units, t.dst_off, rwarp, lane); break;
    case KK_OP_F8E4M3_BF16: consume_f8<F16, false>(D, pay, t.n_units, t.dst_off, ctid); break;
    case KK_OP_F8E5M2_BF16: consume_f8<F16, true>(D, pay, t.n_units, t.dst_off, ctid); break;
    case KK_OP_T_F32_BF16: run_t<F16, 4, 1>(D, L.src, t, sbase, ctid); break;
    case KK_OP_T_F16_BF16: run_t<F16, 2, 2>(D, L.src, t, sbase, ctid); break;
    case KK_OP_T_B16: run_t<F16, 2, 0>(D, L.src, t, sbase, ctid); break;
    case KK_OP_T_B32: run_t<F16, 4, 3>(D, L.src, t, sbase, ctid); break;
    default: break;
  }
}
