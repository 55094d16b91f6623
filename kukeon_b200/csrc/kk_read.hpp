// Read path of the staging pipeline (host only, no CUDA): a chunk's file ranges from the page cache into its pinned staging slot.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "kk_plan.hpp"

namespace kk {

struct FdSet {
  enum MapPolicy { kMapNone = 0, kMapTmpfs, kMapAll };  // which shards get a read-only mapping next to their descriptor
  std::vector<int> fds;
  std::vector<const uint8_t*> maps;  // read-only mappings (nullptr = none): long ranges are copied out of them with streaming stores, see read_chunk
  std::vector<uint64_t> sizes;
  explicit FdSet(const std::vector<std::string>& paths, MapPolicy policy = kMapNone);
  // Bytes of shard i that may be read through its mapping right now: touching a mapped page past the end of a file that has been truncated since
  // it was mapped raises SIGBUS, where pread reports a short read.  Asked once per chunk (one fstat per 16 MiB), this narrows that window from the
  // whole load to one chunk's copy; a range beyond the returned size takes the pread path and its KK_EIO.
  uint64_t live_size(uint32_t i) const;
  void cleanup();
  ~FdSet() { cleanup(); }
  FdSet(const FdSet&) = delete;
  FdSet& operator=(const FdSet&) = delete;
};

void pread_full(int fd, uint8_t* dst, uint64_t len, uint64_t off, const std::string& name);

// KUKEON_GPULOAD_READ = pread (never map) | mapped (map every shard, whatever the file system); unset: map shards on tmpfs.  Measurement knob, not API.
enum ReadMode { kReadAuto = 0, kReadPread, kReadMapped };
ReadMode read_mode();
FdSet::MapPolicy map_policy();

// Copy with streaming stores where the CPU has them (AVX2); the stores are globally visible when it returns.
void copy_nt(uint8_t* dst, const uint8_t* src, size_t n);

// Fill the slot with the chunk's file bytes.
void read_chunk(const Chunk& c, const FdSet& fds, const Index& ix, uint8_t* pinned);

}  // namespace kk
