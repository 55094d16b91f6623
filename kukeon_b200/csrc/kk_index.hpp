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
  uint64_t n_elems() const {
    uint64_t n = 1;
    for (auto d : shape) n *= d;
    return n;
  }
};

struct Index {
  std::string format;               // "safetensors" | "gguf"
  std::vector<std::string> shards;  // absolute paths
  std::vector<uint64_t> shard_bytes;
  std::vector<TensorRec> tensors;   // sorted by (shard, file_offset, name)
  // select_layers (kk_plan.hpp): the tensors are the pipeline stage [layer_begin, layer_end) of a checkpoint of n_layers layers.
  // layer_end == 0: the whole checkpoint.
  uint32_t layer_begin = 0, layer_end = 0;
  uint64_t n_layers = 0;
};

// Throws kk::Error.
Index index_path(const std::string& path);

// Exposed for tests of the individual parsers.
void index_safetensors_file(const std::string& file, uint32_t shard, std::vector<TensorRec>& out, uint64_t* file_bytes);
void index_gguf_file(const std::string& file, uint32_t shard, std::vector<TensorRec>& out, uint64_t* file_bytes);

}  // namespace kk
