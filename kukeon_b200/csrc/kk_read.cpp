#include "kk_read.hpp"

#include <fcntl.h>
#if defined(__x86_64__)
#include <immintrin.h>
#endif
#include <sys/mman.h>
#include <sys/stat.h>
#include <sys/vfs.h>
#include <unistd.h>

#include <algorithm>
#include <cerrno>
#include <cstring>

namespace kk {

FdSet::FdSet(const std::vector<std::string>& paths, MapPolicy policy) {
  for (auto& p : paths) {
    int fd = ::open(p.c_str(), O_RDONLY | O_CLOEXEC);
    if (fd < 0) {
      int e = errno;
      cleanup();
      fail(e == ENOENT ? KK_ENOENT : KK_EIO, "open %s: %s", p.c_str(), strerror(e));
    }
    fds.push_back(fd);
    const uint8_t* mp = nullptr;
    uint64_t sz = 0;
    bool want = policy == kMapAll;
    if (policy == kMapTmpfs) {
      struct statfs sf;
      want = fstatfs(fd, &sf) == 0 && (unsigned long)sf.f_type == 0x01021994ul;  // TMPFS_MAGIC: every byte is in memory, a mapping never waits for a disk
    }
    if (want) {
      struct stat st;
      if (fstat(fd, &st) == 0 && st.st_size > 0) {
        void* m = mmap(nullptr, (size_t)st.st_size, PROT_READ, MAP_SHARED, fd, 0);
        if (m != MAP_FAILED) { mp = (const uint8_t*)m; sz = (uint64_t)st.st_size; }
      }
    }
    maps.push_back(mp);
    sizes.push_back(sz);
  }
}

uint64_t FdSet::live_size(uint32_t i) const {
  struct stat st;
  if (fstat(fds[i], &st) != 0 || st.st_size < 0) return 0;
  return std::min<uint64_t>((uint64_t)st.st_size, sizes[i]);
}

void FdSet::cleanup() {
  for (size_t i = 0; i < maps.size(); ++i)
    if (maps[i]) munmap((void*)maps[i], sizes[i]);
  for (int f : fds) ::close(f);
  maps.clear();
  fds.clear();
}

void pread_full(int fd, uint8_t* dst, uint64_t len, uint64_t off, const std::string& name) {
  while (len) {
    ssize_t r = ::pread(fd, dst, len > (1ull << 30) ? (1ull << 30) : len, (off_t)off);
    if (r < 0) {
      if (errno == EINTR) continue;
      fail(KK_EIO, "pread %s @%llu: %s", name.c_str(), (unsigned long long)off, strerror(errno));
    }
    if (r == 0) fail(KK_EIO, "pread %s @%llu: unexpected end of file", name.c_str(), (unsigned long long)off);
    dst += r;
    off += (uint64_t)r;
    len -= (uint64_t)r;
  }
}

// How a chunk's long contiguous ranges travel from the page cache into the pinned slot (Llama-3-8B from tmpfs, 16 reader threads):
//   pread                       the kernel's copy_to_user, 4 KiB at a time: the load is reader-bound
//   mapping + memcpy            no faster than pread, and the final munmap of a checkpoint-sized mapping is ONE thread tearing down 4 M page-table
//                               entries
//   mapping + streaming stores  about half pread's copy time per thread (no read-for-ownership of the slot's lines, which only the DMA engine
//                               reads next) — with the same munmap bill
//   ... + MADV_DONTNEED of each range right after its copy (the reader threads drop their own page-table entries in parallel, the final munmap
//                               finds none): the load becomes H2D-bound.  DEFAULT for shards on tmpfs; other file systems keep pread (a mapping of
//                               a cold file would fault page by page into the disk).
//   MAP_POPULATE mapping per range: slower than pread (every mmap / munmap takes the process's mm lock exclusively).
//   cache-resident bounce ring (4 x 256 KiB pinned pieces per reader between mapping and device slot, so that neither the CPU's stores nor the copy
//                               engine's reads reach DRAM): faster CPU copy, but 64 K small H2D copies starve the copy engines.
// The slower forms are deleted (git history: ed69c4b..50a97f8 carry them); what is left is the default and one switch, KUKEON_GPULOAD_READ.
ReadMode read_mode() {
  static const ReadMode mode = [] {
    const char* e = getenv("KUKEON_GPULOAD_READ");
    if (!e) return kReadAuto;
    if (!strcmp(e, "pread")) return kReadPread;
    if (!strcmp(e, "mapped")) return kReadMapped;
    return kReadAuto;
  }();
  return mode;
}

FdSet::MapPolicy map_policy() {
  switch (read_mode()) {
    case kReadAuto: return FdSet::kMapTmpfs;
    case kReadPread: return FdSet::kMapNone;
    default: return FdSet::kMapAll;
  }
}

#if defined(__x86_64__)
__attribute__((target("avx2"))) static void copy_nt_avx2(uint8_t* dst, const uint8_t* src, size_t n) {
  size_t head = (32u - ((uintptr_t)dst & 31u)) & 31u;
  if (head > n) head = n;
  if (head) { memcpy(dst, src, head); dst += head; src += head; n -= head; }
  size_t i = 0;
  for (; i + 128 <= n; i += 128) {
    const __m256i a = _mm256_loadu_si256((const __m256i*)(src + i)), b = _mm256_loadu_si256((const __m256i*)(src + i + 32));
    const __m256i c = _mm256_loadu_si256((const __m256i*)(src + i + 64)), d = _mm256_loadu_si256((const __m256i*)(src + i + 96));
    _mm256_stream_si256((__m256i*)(dst + i), a);
    _mm256_stream_si256((__m256i*)(dst + i + 32), b);
    _mm256_stream_si256((__m256i*)(dst + i + 64), c);
    _mm256_stream_si256((__m256i*)(dst + i + 96), d);
  }
  if (i < n) memcpy(dst + i, src + i, n - i);
  _mm_sfence();  // the streaming stores must be globally visible before the H2D copy of the slot is enqueued
}
#endif
void copy_nt(uint8_t* dst, const uint8_t* src, size_t n) {
#if defined(__x86_64__)
  static const bool avx2 = __builtin_cpu_supports("avx2");
  if (avx2) { copy_nt_avx2(dst, src, n); return; }
#endif
  memcpy(dst, src, n);
}

void read_chunk(const Chunk& c, const FdSet& fds, const Index& ix, uint8_t* pinned) {
  static const uint64_t pg = (uint64_t)sysconf(_SC_PAGESIZE);
  const uint8_t* mp = fds.maps.empty() ? nullptr : fds.maps[c.shard];
  const uint64_t msz = mp ? fds.live_size(c.shard) : 0;
  const ReadMode mode = read_mode();
  for (auto& r : c.reads) {
    const bool in_map = mp && r.file_off <= msz && r.len <= msz - r.file_off;  // (a file that shrank since it was mapped takes pread's error path)
    if (in_map && r.len > (256u << 10) && mode != kReadPread) {
      copy_nt(pinned + r.buf_off, mp + r.file_off, r.len);
      const uint64_t a = (r.file_off + pg - 1) & ~(pg - 1), e = (r.file_off + r.len) & ~(pg - 1);  // the whole pages inside the range
      if (e > a) madvise((void*)(mp + a), (size_t)(e - a), MADV_DONTNEED);  // page-table entries only: the pages stay in the page cache
      continue;
    }
    // short ranges (column-slice rows of a SCATTER load: thousands of 2-7 KB runs per chunk) stay on pread: copied out of the mapping the 70B
    // scatter load is slower — a first-touch page fault per row costs more than the syscall
    pread_full(fds.fds[c.shard], pinned + r.buf_off, r.len, r.file_off, ix.shards[c.shard]);
  }
}

}  // namespace kk
