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

// JSON description of a plan (kk_plan_describe).
std::string plan_to_json(const Plan& P);

// How a load moves its bytes between the devices.
enum class LoadOrder {
  kOwn,       // every local device converts its own plan part into its own pool, and nothing else (SINGLE, SCATTER, BROADCAST with no peer)
  kReplicas,  // BROADCAST, one process, >= 2 devices that do not store into each other (KK_FANOUT_NONE, or no peer access): each converts every part
  kPush,      // BROADCAST, KK_FANOUT_P2P: the convert kernel also stores into every other pool (the context's, or the attached ranks')
  kNvls,      // BROADCAST, KK_FANOUT_NVLS: one multimem.st per vector through the multicast object the pools are bound to
  kRaw,       // BROADCAST, KK_FANOUT_RAW: file bytes all-gathered into per-device raw images (stage 1), each converted locally (stage 2)
  kPull,      // BROADCAST, KK_FANOUT_PULL: own part into the own pool and a slice buffer (stage 1), the peers' slices pulled in (stage 2)
};

// A load's options resolved against its context, once per model: every stage of the load switches on this.
struct LoadShape {
  LoadOrder order = LoadOrder::kOwn;
  bool multi_proc = false;       // one rank of a one-process-per-GPU load (part_count > 1)
  int rank = 0;                  // the plan part this process ingests when multi_proc, else 0
  int n_parts = 1;               // plan parts: 1 for SINGLE, else the ranks or the context's devices
  std::vector<int> local_parts;  // per local device li (context device li): the plan part it ingests
  bool every_part = false;       // every local device converts every plan part: kReplicas, and kNvls without peer access
  bool xdst = false;             // the scatter row exchange: every launch carries every rank's pool (ConvertLaunch::xdst)
  bool peer_ok = false;          // the context's devices reach each other's memory
  bool two_stage = false;        // loaded only once kk_convert_local has run (multi-process RAW and PULL)
};

// Validates opts against a context of n_devices devices (peer_ok: with peer access between all of them) and resolves the load's shape;
// throws KK_EINVAL / KK_EUNSUPPORTED.  The checks that need the driver (NVLS support) or the plan (multimem, PULL's pool ranges) and
// RAW's need for peer access (checked when stage 1 runs) stay with the load.
LoadShape resolve_load_shape(const kk_load_opts& opts, int n_devices, bool peer_ok);

// Pool bytes from s.dst_off on that segment s spans in each destination pool.  Copies, casts and block dequantisers fill that range; a
// transpose spans its whole output tensor but stores only its own rows' columns of it, strided; KK_OP_ROWSPLIT spans nothing here (its
// rows land in every rank's pool).
uint64_t seg_out_extent(const KKSeg& s);

}  // namespace kk
