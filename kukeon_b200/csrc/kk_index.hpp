// Checkpoint indexing ("Pull"): safetensors (single / sharded with index.json) and GGUF v2/v3.
// CPU only. Produces the tensor index SURVEY.md §8(a2) defines:
//   (name, dtype, shape outermost-first, shard, absolute file offset, nbytes) sorted by (shard, offset).
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "kk_common.hpp"

namespace kk {

struct TensorRec {
  std::string name;
  uint32_t dtype = 0;
  std::vector<uint64_t> shape;
  uint32_t shard = 0;
  uint64_t file_offset = 0;
  uint64_t nbytes = 0;
  // to_hf_layout: llama.cpp interleaved the two rotary halves of each of this many heads in the rows (0: rows as in the file)
  uint32_t rope_heads = 0;
  uint64_t n_elems() const {
    uint64_t n = 1;
    for (auto d : shape) n *= d;
    return n;
  }
};

// One GGUF metadata value, recorded as the file has it.  Indexing never fails on these: a load that needs the value (to_hf_layout)
// raises err with why, or KK_EFORMAT when the key is missing.
struct GgufKey {
  bool seen = false;  // the key is in the file
  int err = 0;        // seen: 0 when the value is usable, else KK_EFORMAT (ill-typed, out of range) or KK_EUNSUPPORTED (a per-layer array)
  std::string why;
  uint64_t u = 0;     // integer keys: 1..65535
  std::string s;      // string keys
  bool operator==(const GgufKey& o) const { return seen == o.seen && err == o.err && u == o.u && s == o.s; }
};

// The GGUF metadata the HF view (KK_LOAD_HF_LAYOUT) reads.  <arch> is general.architecture.
struct GgufMeta {
  GgufKey arch;           // general.architecture
  GgufKey head_count;     // <arch>.attention.head_count
  GgufKey head_count_kv;  // <arch>.attention.head_count_kv (absent for MHA models: then head_count)
  GgufKey expert_count;   // <arch>.expert_count
};

struct Index {
  std::string format;               // "safetensors" | "gguf"
  GgufMeta gguf;                    // GGUF: from the first shard (a later shard that repeats a key and disagrees marks it bad)
  std::string hf_arch;              // to_hf_layout: the tensors are the HF view of a checkpoint of this architecture
  std::vector<std::string> shards;  // absolute paths
  std::vector<uint64_t> shard_bytes;
  std::vector<TensorRec> tensors;   // sorted by (shard, file_offset, name)
  // select_layers: the tensors are the pipeline stage [layer_begin, layer_end) of a checkpoint of n_layers layers.
  // layer_end == 0: the whole checkpoint.
  uint32_t layer_begin = 0, layer_end = 0;
  uint64_t n_layers = 0;
};

// Throws kk::Error.
Index index_path(const std::string& path);

// Exposed for tests of the individual parsers.
void index_safetensors_file(const std::string& file, uint32_t shard, std::vector<TensorRec>& out, uint64_t* file_bytes);
void index_gguf_file(const std::string& file, uint32_t shard, std::vector<TensorRec>& out, uint64_t* file_bytes, GgufMeta* meta = nullptr);

// Pipeline stage [layer_begin, layer_end) of a checkpoint (the rule is documented next to kk_load_opts in kukeon_gpuload.h).  Keeps the
// shard list, every kept record's shard index and the index order; layer_end == 0 with layer_begin == 0 returns the index unchanged.
// Throws KK_EINVAL (empty or out-of-range range) and KK_EUNSUPPORTED (no layered tensors, or two numbered stacks).
Index select_layers(Index index, uint32_t layer_begin, uint32_t layer_end);

// The Hugging Face view of a GGUF checkpoint under KK_LOAD_HF_LAYOUT (the rule is documented next to the flag in kukeon_gpuload.h); any
// other flags return the index unchanged.  Renames every tensor, splits each expert stack into one record per expert (a byte range of the
// stack) and marks llama's Q/K tensors (TensorRec::rope_heads) for build_plan to un-permute; the index order stays (shard, file offset).
// Throws KK_EINVAL (not a GGUF checkpoint), KK_EFORMAT (a needed metadata key missing or ill-typed, Q/K rows not a multiple of 2 * heads)
// and KK_EUNSUPPORTED (an architecture or a tensor outside the table).  Runs before select_layers.
Index to_hf_layout(Index index, uint32_t flags);

// The index a load plans over: the checkpoint at path, in its Hugging Face view under KK_LOAD_HF_LAYOUT, then cut to the pipeline
// stage [layer_begin, layer_end).  Throws what index_path, to_hf_layout and select_layers throw.
Index index_for_load(const std::string& path, uint32_t flags, uint32_t layer_begin, uint32_t layer_end);

}  // namespace kk
