// Host test of the loader's page-cache -> staging-slot read paths (kk_read.cpp: FdSet, read_chunk, copy_nt) — test infrastructure only.
// Linked against kk_read.o alone; no CUDA (no GPU needed).  Usage:
//   KUKEON_GPULOAD_READ=<mode> kk_read_test <dir> <policy: none|tmpfs|all> [seed of the random chunks]
// Writes a pseudo-random file into <dir>, fills a poisoned buffer through read_chunk with a mix of long (> 256 KiB, unaligned) and short ranges,
// compares every range with the file and every byte outside the ranges with the poison, and prints one JSON line.
#include "kk_read.hpp"

#include <unistd.h>

#include <cstdio>
#include <cstring>
#include <random>

using namespace kk;

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  const std::string dir = argv[1], pol = argv[2];
  const std::string path = dir + "/read_test.bin";
  const size_t fsz = 5u * 1024u * 1024u + 12345u;
  std::vector<uint8_t> file(fsz);
  std::mt19937_64 rng(42);
  for (size_t i = 0; i + 8 <= fsz; i += 8) { uint64_t v = rng(); memcpy(&file[i], &v, 8); }
  FILE* f = fopen(path.c_str(), "wb");
  if (!f || fwrite(file.data(), 1, fsz, f) != fsz) return 3;
  fclose(f);
  int bad = 0, mapped = 0;
  std::string err;
  try {
    Index ix;
    ix.shards.push_back(path);
    FdSet fds(ix.shards, pol == "all" ? FdSet::kMapAll : pol == "tmpfs" ? FdSet::kMapTmpfs : FdSet::kMapNone);
    mapped = fds.maps[0] != nullptr;
    // ranges: (file_off, len) — long ones off page and 32-byte boundaries, short ones, one ending at the last byte of the file
    const std::vector<std::pair<uint64_t, uint64_t>> want = {{3, 1000003}, {1000100, 7}, {1000200, 300 * 1024 + 1}, {1400000, 4096}, {1500001, 262144}, {1800007, 262145},
                                                            {2200000, 2 * 1024 * 1024 + 33}, {fsz - 600000, 600000}};
    Chunk c;
    c.shard = 0;
    uint64_t pos = 0;
    for (auto& w : want) {
      const uint64_t at = (pos + 15) & ~15ull;
      c.reads.push_back({w.first, w.second, at});
      pos = at + w.second;
    }
    c.buf_bytes = pos;
    std::vector<uint8_t> buf(pos + 64, 0xA5);
    uint8_t* dst = buf.data() + 1;  // an odd destination: the streaming copy has to find its own 32-byte boundary
    read_chunk(c, fds, ix, dst);
    std::vector<uint8_t> covered(pos + 64, 0);
    for (auto& r : c.reads) {
      if (memcmp(dst + r.buf_off, file.data() + r.file_off, r.len)) ++bad;
      for (uint64_t i = 0; i < r.len; ++i) covered[1 + r.buf_off + i] = 1;
    }
    for (size_t i = 0; i < buf.size(); ++i)
      if (!covered[i] && buf[i] != 0xA5) { ++bad; break; }
    // the mapping must still serve reads after the per-range MADV_DONTNEED (pages stay in the page cache): read everything again
    read_chunk(c, fds, ix, dst);
    for (auto& r : c.reads)
      if (memcmp(dst + r.buf_off, file.data() + r.file_off, r.len)) ++bad;
    // a range past the end of the file is refused with KK_EIO whatever the mode
    Chunk over;
    over.shard = 0;
    over.reads.push_back({fsz - 100, 300 * 1024, 0});
    try {
      read_chunk(over, fds, ix, dst);
      ++bad;
    } catch (const Error& e) {
      if (e.code != KK_EIO) ++bad;
    }
    // seeded random chunks: ranges of 1 B .. 2 MiB at arbitrary file offsets, 16-byte aligned buffer offsets as the planner lays them out
    {
      std::mt19937_64 r2(argc > 3 ? strtoull(argv[3], nullptr, 10) : 7);
      for (int round = 0; round < 6; ++round) {
        Chunk rc;
        rc.shard = 0;
        uint64_t p2 = 0;
        const int n = 1 + (int)(r2() % 24);
        for (int i = 0; i < n; ++i) {
          const uint64_t len = (r2() % 4 == 0) ? 1 + r2() % 300 : 1 + r2() % (2u << 20);
          const uint64_t off = r2() % (fsz - len);
          const uint64_t at = (p2 + 15) & ~15ull;
          rc.reads.push_back({off, len, at});
          p2 = at + len;
        }
        rc.buf_bytes = p2;
        std::vector<uint8_t> b2(p2 + 64, 0x5A);
        uint8_t* d2 = b2.data() + (r2() % 32);
        read_chunk(rc, fds, ix, d2);
        for (auto& r : rc.reads)
          if (memcmp(d2 + r.buf_off, file.data() + r.file_off, r.len)) ++bad;
        if (b2[p2 + 63] != 0x5A) ++bad;
      }
    }
    // a shard truncated AFTER it was mapped: the chunk's ranges beyond the new end must come back as KK_EIO (pread's short read), not as a SIGBUS
    if (truncate(path.c_str(), 1200000) != 0) ++bad;
    Chunk late;
    late.shard = 0;
    late.reads.push_back({1000200, 300 * 1024 + 1, 0});
    try {
      read_chunk(late, fds, ix, dst);
      ++bad;
    } catch (const Error& e) {
      if (e.code != KK_EIO) ++bad;
    }
    Chunk early;  // what is still inside the file keeps working
    early.shard = 0;
    early.reads.push_back({3, 1000003, 0});
    read_chunk(early, fds, ix, dst);
    if (memcmp(dst, file.data() + 3, 1000003)) ++bad;
  } catch (const Error& e) {
    err = e.what();
    ++bad;
  }
  unlink(path.c_str());
  printf("{\"bad\":%d,\"mapped\":%d,\"mode\":%d,\"error\":\"%s\"}\n", bad, mapped, (int)read_mode(), err.c_str());
  return bad ? 1 : 0;
}
