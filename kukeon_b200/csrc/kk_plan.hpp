// Load planning (host, no CUDA): pool layout, per-rank chunk lists, segment tables.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "kk_index.hpp"
#include "kk_ops.h"

namespace kk {

constexpr uint32_t kNoSlice = 0xFFFFFFFFu;

struct Placement {
  uint32_t dtype = 0;            // dtype in the pool
  std::vector<uint64_t> shape;   // shape in the pool (after transpose / slice)
  uint64_t pool_offset = 0;
  uint64_t nbytes = 0;
  uint32_t slice_dim = kNoSlice;
  uint64_t slice_begin = 0;
};

struct ReadOp {
  uint64_t file_off;
  uint64_t len;
  uint64_t buf_off;  // where in the chunk's staging buffer the bytes land
};

struct Chunk {
  uint32_t shard = 0;
  std::vector<ReadOp> reads;
  uint64_t buf_bytes = 0;   // staging bytes used (without the 16-B over-read slack)
  uint32_t seg_begin = 0;   // into PartPlan::segs; seg.src_off is relative to the chunk buffer,
  uint32_t seg_count = 0;   // seg.tile_begin relative to the chunk's first tile
  uint32_t n_tiles = 0;
  uint64_t src_bytes = 0;   // file bytes this chunk reads
  uint64_t out_bytes = 0;   // pool bytes it produces (per destination)
};

struct PartPlan {
  std::vector<Chunk> chunks;
  std::vector<KKSeg> segs;
  uint64_t src_bytes = 0;
  uint64_t out_bytes = 0;
};

struct Plan {
  Index index;
  int mode = 0;
  uint32_t flags = 0;
  int n_parts = 1;
  // SINGLE/BROADCAST: placements[0] applies to every device. SCATTER: placements[part].
  std::vector<std::vector<Placement>> placements;
  std::vector<uint64_t> pool_bytes;  // same indexing as placements
  std::vector<PartPlan> parts;       // one per ingesting rank/device
  uint64_t file_bytes = 0;           // sum of tensor bytes in the files
  const std::vector<Placement>& placement_of_part(int part) const {
    return placements.size() == 1 ? placements[0] : placements[(size_t)part];
  }
  uint64_t pool_bytes_of_part(int part) const { return pool_bytes.size() == 1 ? pool_bytes[0] : pool_bytes[(size_t)part]; }
};

// chunk_bytes: staging slot size (upper bound on Chunk::buf_bytes).
Plan build_plan(Index index, int mode, uint32_t flags, int n_parts, uint64_t chunk_bytes);

// Which dimension a tensor is sliced along in SCATTER mode (kNoSlice = replicate). [PROPOSED] rule of
// SURVEY.md §8(a3.S5): column-parallel weights along dim 0, row-parallel weights along dim 1.
uint32_t scatter_slice_dim(const TensorRec& t, int n_parts);

// JSON description of a plan (kk_plan_describe).
std::string plan_to_json(const Plan& P);

// True when KK_LOAD_GPT2_CONV1D_T applies to this tensor.
bool is_gpt2_conv1d(const TensorRec& t);

// Pool bytes from s.dst_off on that segment s spans in each destination pool.  Copies, casts and block dequantisers fill that range; a
// transpose spans its whole output tensor but stores only its own rows' columns of it, strided; KK_OP_ROWSPLIT spans nothing here (its
// rows land in every rank's pool).
uint64_t seg_out_extent(const KKSeg& s);

}  // namespace kk
