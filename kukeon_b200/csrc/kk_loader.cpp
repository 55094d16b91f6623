// Host side of the loader: staging pipeline (page cache -> pinned ring -> H2D -> convert/fan-out kernel),
// pool allocation, refcounted model registry, IPC export, resident-image measurement mode.
//
// Pipeline per ingesting device (SURVEY.md §8(a3.S2-S4)), stream_part:
//   R reader threads, each with its own CUDA stream and >= 2 pinned slots (+ matching device staging
//   buffers).  A thread claims the next chunk, waits for its slot's previous work (event), reads the
//   chunk's file ranges into the pinned slot (kk_read.cpp), enqueues what moves the chunk on (H2D, launches) on its stream and moves
//   on.  Disk/page-cache reads, PCIe DMA and the kernels of different threads overlap.  In a streaming load the convert kernel writes
//   bf16 into the local pool and, in BROADCAST mode, into every peer pool over NVLink in the same pass.
#include "kk_loader.hpp"

#include <pthread.h>
#include <sched.h>

#include <algorithm>
#include <chrono>
#include <cstring>
#include <exception>
#include <sstream>
#include <thread>

#include "kk_json.hpp"
#include "kk_lora.cuh"
#include "kk_read.hpp"

namespace kk {

namespace {

double now_s() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// CPUs of the NUMA node the device hangs off (empty when sysfs does not say).
std::vector<int> numa_cpus_of_device(int ordinal) {
  std::vector<int> cpus;
  char bdf[32] = {0};
  try {
    device_identity(ordinal, bdf, sizeof bdf, nullptr, 0);
  } catch (const Error&) {
    cudaGetLastError();
    return cpus;
  }
  char path[256];
  snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bdf);
  FILE* f = fopen(path, "r");
  if (!f) return cpus;
  int node = -1;
  if (fscanf(f, "%d", &node) != 1) node = -1;
  fclose(f);
  if (node < 0) return cpus;
  snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
  f = fopen(path, "r");
  if (!f) return cpus;
  char buf[4096] = {0};
  if (fgets(buf, sizeof buf, f)) {
    char* save = nullptr;  // strtok_r: kk_open may run on several threads at once
    for (char* tok = strtok_r(buf, ",\n", &save); tok; tok = strtok_r(nullptr, ",\n", &save)) {
      int a, b;
      if (sscanf(tok, "%d-%d", &a, &b) == 2) { for (int i = a; i <= b; ++i) cpus.push_back(i); }
      else if (sscanf(tok, "%d", &a) == 1) cpus.push_back(a);
    }
  }
  fclose(f);
  return cpus;
}

void pin_this_thread(const std::vector<int>& cpus) {
  if (cpus.empty()) return;
  cpu_set_t set;
  CPU_ZERO(&set);
  for (int c : cpus)
    if (c >= 0 && c < CPU_SETSIZE) CPU_SET(c, &set);
  pthread_setaffinity_np(pthread_self(), sizeof set, &set);  // best effort
}

struct ErrorSink {
  std::mutex mu;
  std::exception_ptr first;
  std::atomic<bool> stop{false};
  void capture() {
    std::lock_guard<std::mutex> g(mu);
    if (!first) first = std::current_exception();
    stop = true;
  }
  void rethrow() {
    if (first) std::rethrow_exception(first);
  }
};

// Device copy of a segment table on device `ordinal` (empty for an empty table).
DevBuf upload_segs(int ordinal, const std::vector<KKSeg>& segs) {
  if (segs.empty()) return DevBuf();
  DevBuf d(ordinal, segs.size() * sizeof(KKSeg), "a segment table");
  KK_CUDA(cudaMemcpy(d.get(), segs.data(), segs.size() * sizeof(KKSeg), cudaMemcpyHostToDevice));
  return d;
}

uint64_t seg_base_of(const Plan& P, int part) {
  uint64_t b = 0;
  for (int i = 0; i < part; ++i) b += P.parts[(size_t)i].segs.size();
  return b;
}

// The chunk buffers of plan parts laid out back to back in one device image, and their segments rebased onto it.
struct ImageLayout {
  std::vector<std::vector<uint64_t>> chunk_off;  // [i][ci]: offset of chunk ci of parts[i] in the image
  uint64_t bytes = 0;
  std::vector<KKSeg> segs;                       // src_off rebased onto the image, tile_begin onto the segment's launch
  std::vector<ImageLaunch> launches;
};

// Every chunk takes its staging bytes plus 64 bytes of over-read slack, at a 256-byte boundary.  One launch per shard, split only where a
// launch would exceed kMaxSegsPerLaunch segments or 0xFFFFFFF0 tiles: kk_convert_resident reports one time per launch.
ImageLayout lay_out_image(const Plan& P, const std::vector<int>& parts) {
  ImageLayout im;
  int last_shard = -1;
  for (int part : parts) {
    const PartPlan& pp = P.parts[(size_t)part];
    im.chunk_off.emplace_back();
    for (const Chunk& ch : pp.chunks) {
      const uint64_t off = im.bytes;
      im.chunk_off.back().push_back(off);
      im.bytes += align_up(ch.buf_bytes + 64, 256);
      if (im.launches.empty() || last_shard != (int)ch.shard || im.launches.back().n_segs + ch.seg_count > kMaxSegsPerLaunch ||
          (uint64_t)im.launches.back().n_tiles + ch.n_tiles > 0xFFFFFFF0ull)
        im.launches.push_back({(uint32_t)im.segs.size(), 0, 0});
      last_shard = (int)ch.shard;
      ImageLaunch& L = im.launches.back();
      for (uint32_t j = 0; j < ch.seg_count; ++j) {
        KKSeg sg = pp.segs[ch.seg_begin + j];
        sg.src_off += off;
        sg.tile_begin += L.n_tiles;
        im.segs.push_back(sg);
      }
      L.n_segs += ch.seg_count;
      L.n_tiles += ch.n_tiles;
    }
  }
  return im;
}

// Test hook: KUKEON_GPULOAD_TEST_NDST=<n> pads the destination list to n entries by repeating the ones it has,
// so that the kernel's n-destination store paths (the 8-GPU fan-out ladder) can be exercised on a box with fewer
// GPUs.  Writing the same bytes to the same pool several times is harmless.
void pad_dsts_for_test(ConvertLaunch& L) {
  static const int want = [] {
    const char* e = getenv("KUKEON_GPULOAD_TEST_NDST");
    return e ? atoi(e) : 0;
  }();
  if (want <= 0) return;
  const uint32_t have = L.n_dst;
  while (L.n_dst < (uint32_t)want && L.n_dst < KK_MAX_DST) { L.dst[L.n_dst] = L.dst[L.n_dst % have]; L.n_dst++; }
}

// multimem.st exists for 4-, 8- and 16-byte accesses only: a plan qualifies for KK_LAUNCH_MULTIMEM when no segment ever needs a 1- or
// 2-byte store — every tile of it is whole 16-byte output vectors.  Transposes store single elements at tile edges and are excluded; FP8
// widening works on 16-element groups and needs whole groups.
bool plan_allows_multimem(const Plan& P, std::string* why) {
  for (auto& pp : P.parts)
    for (auto& s : pp.segs) {
      const bool f8 = s.op == KK_OP_F8E4M3_BF16 || s.op == KK_OP_F8E5M2_BF16;
      if (kk_is_transpose(s.op) || s.op == KK_OP_ROWSPLIT || seg_out_extent(s) % 16 != 0 || (f8 && s.units % 16 != 0)) {
        if (why) *why = "a tensor's size is not a whole number of 16-byte output vectors (or the load transposes); multimem.st cannot store its tail";
        return false;
      }
    }
  return true;
}

// Pool bytes [lo, hi) that plan part `part` produces, KK_OP_ROWSPLIT segments left out (their rows land in every rank's pool).  Pool
// order equals file order, so for every op that writes its output linearly this is one contiguous range and the ranges of different
// parts are disjoint.  Returns false when the part carries ops whose output is not linear in the pool (the scatter row exchange;
// transposes, whose strided stores interleave with the other parts' inside the tensor-wide extent counted here): such plans cannot be
// pulled slice by slice.
bool part_pool_range(const Plan& P, int part, uint64_t& lo, uint64_t& hi) {
  lo = UINT64_MAX;
  hi = 0;
  bool linear = true;
  for (auto& s : P.parts[(size_t)part].segs) {
    if (s.op == KK_OP_ROWSPLIT) { linear = false; continue; }
    if (kk_is_transpose(s.op)) linear = false;
    lo = std::min(lo, s.dst_off);
    hi = std::max(hi, s.dst_off + seg_out_extent(s));
  }
  if (lo == UINT64_MAX) lo = 0;
  return linear;
}

// The output format of m's convert launches: KK_LAUNCH_F16 for a KK_LOAD_F16 model, which launch_convert runs on the fp16 kernel.
uint32_t format_flags(const kk_model* m) { return (m->plan.flags & KK_LOAD_F16) ? KK_LAUNCH_F16 : 0u; }

// Destination pools a convert launch on local device `li` writes to, and the launch's output format.
void fill_dsts(kk_model* m, int li, ConvertLaunch& L) {
  const LoadShape& S = m->shape;
  L.n_dst = 0;
  L.flags = format_flags(m);
  for (auto& d : L.dst) d = nullptr;
  L.dst[L.n_dst++] = m->pools[(size_t)li].ptr;
  L.n_xdst = 0;
  for (auto& d : L.xdst) d = nullptr;
  if (S.xdst) {
    // all-to-all destinations of KK_OP_ROWSPLIT segments: the pool of every rank, indexed by rank
    for (int j = 0; j < S.n_parts; ++j) {
      uint8_t* p = nullptr;
      if (S.multi_proc) p = (j == S.rank) ? m->pools[0].ptr : (uint8_t*)m->peer[kPeerPool][j].ptr;
      else if (S.peer_ok) p = m->pools[(size_t)j].ptr;
      if (!p) fail(KK_ESTATE, "KK_LOAD_SCATTER_EXCHANGE: the pool of rank %d is not reachable (attach it with kk_peer_attach, or enable peer access)", j);
      L.xdst[j] = p;
    }
    L.n_xdst = (uint32_t)S.n_parts;
  }
  switch (S.order) {
    case LoadOrder::kNvls:  // one multimem.st per vector reaches every pool through the switch
      L.dst[0] = m->nvls->multicast();
      L.n_dst = 1;
      L.flags |= KK_LAUNCH_MULTIMEM;
      return;
    case LoadOrder::kPull:  // stage 1 of a pull load: the same bytes into the slice buffer the peers will read (pool offset -> slice_buf - slice_base)
      if (m->slice_buf) L.dst[L.n_dst++] = (uint8_t*)((uintptr_t)m->slice_buf.get() - (uintptr_t)m->slice_base);
      return;
    case LoadOrder::kPush:
      if (S.multi_proc) {
        for (auto& b : m->peer[kPeerPool])
          if (b.ptr) L.dst[L.n_dst++] = (uint8_t*)b.ptr;
      } else {
        for (size_t j = 0; j < m->pools.size(); ++j)
          if ((int)j != li) L.dst[L.n_dst++] = m->pools[j].ptr;
      }
      break;
    default:  // the own pool alone (a RAW model converts through convert_local_all)
      break;
  }
  pad_dsts_for_test(L);
}

// Peer raw images a stage-1 copy launch on local device li writes to (never the local image: it is the source).
void fill_raw_dsts(kk_model* m, int li, ConvertLaunch& L) {
  L.n_dst = 0;
  L.flags = format_flags(m);
  for (auto& d : L.dst) d = nullptr;
  if (m->shape.multi_proc) {
    for (auto& b : m->peer[kPeerRaw])
      if (b.ptr) L.dst[L.n_dst++] = (uint8_t*)b.ptr;
  } else {
    for (size_t j = 0; j < m->images.size(); ++j)
      if ((int)j != li) L.dst[L.n_dst++] = m->images[j].image.get();
  }
}

// Stream plan part `part` through the reader threads of local device `li`.  Each thread claims the next chunk, waits until its next slot's
// previous work has run, reads the chunk into the pinned slot and calls consume(reader, slot, chunk index), which enqueues on the reader's
// stream what moves the bytes on; the slot is free again once that has run.  record_times: this is the streaming pass of kk_load_part, whose
// reader timings stats() reports.
template <class Consume>
void stream_part(kk_model* m, int li, int part, const FdSet& fds, bool record_times, const Consume& consume) {
  kk_ctx* c = m->ctx;
  Device& dev = c->devs[(size_t)li];
  const PartPlan& pp = m->plan.parts[(size_t)part];
  std::lock_guard<std::mutex> pipeline(*dev.load_mu);
  std::atomic<size_t> next{0};
  ErrorSink sink;
  auto ns = [] { return (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
  auto worker = [&](Reader* rd) {
    try {
      if (!(c->cfg.flags & KK_CFG_NO_NUMA_PIN)) pin_this_thread(dev.numa_cpus);
      KK_CUDA(cudaSetDevice(dev.ordinal));
      size_t k = 0;
      uint64_t w_ns = 0, p_ns = 0, i_ns = 0;
      for (;;) {
        if (sink.stop) break;
        const size_t ci = next.fetch_add(1);
        if (ci >= pp.chunks.size()) break;
        Slot& s = rd->slots[k++ % rd->slots.size()];
        const uint64_t t0 = ns();
        KK_CUDA(cudaEventSynchronize(s.done));
        const uint64_t t1 = ns();
        read_chunk(pp.chunks[ci], fds, m->plan.index, s.pinned);
        const uint64_t t2 = ns();
        consume(*rd, s, ci);
        KK_CUDA(cudaEventRecord(s.done, rd->stream));
        w_ns += t1 - t0; p_ns += t2 - t1; i_ns += ns() - t2;
      }
      const uint64_t t3 = ns();
      KK_CUDA(cudaStreamSynchronize(rd->stream));
      if (record_times) {
        m->rd_drain_ns += ns() - t3;
        m->rd_wait_ns += w_ns; m->rd_pread_ns += p_ns; m->rd_issue_ns += i_ns;
      }
    } catch (...) {
      sink.capture();
    }
  };
  if (record_times) {
    m->rd_wait_ns = 0; m->rd_pread_ns = 0; m->rd_issue_ns = 0; m->rd_drain_ns = 0;
    m->rd_threads = (uint32_t)dev.readers.size();
  }
  std::vector<std::thread> th;
  // every reader runs on its own (NUMA-pinned) thread; the caller's thread affinity is left alone
  for (size_t r = 0; r < dev.readers.size(); ++r) th.emplace_back(worker, &dev.readers[r]);
  for (auto& t : th) t.join();
  if (sink.first) {
    // leave the streams quiet before reporting
    cudaSetDevice(dev.ordinal);
    for (auto& r : dev.readers) cudaStreamSynchronize(r.stream);
  }
  sink.rethrow();
}

// Streaming load of plan part `part` on local device li: H2D into the slot's device buffer (or zero-copy), then the convert launch.
void convert_part(kk_model* m, int li, int part, const FdSet& fds) {
  const PartPlan& pp = m->plan.parts[(size_t)part];
  if (pp.chunks.empty()) return;
  const int sm_count = m->ctx->devs[(size_t)li].sm_count;
  const bool zerocopy = (m->ctx->cfg.flags & KK_CFG_ZEROCOPY) != 0;
  const KKSeg* d_segs = m->d_segs[(size_t)li].get<KKSeg>() + seg_base_of(m->plan, part);
  ConvertLaunch base{};
  fill_dsts(m, li, base);
  stream_part(m, li, part, fds, true, [&](Reader& rd, Slot& s, size_t ci) {
    const Chunk& ch = pp.chunks[ci];
    ConvertLaunch L = base;
    L.src = s.pinned;
    if (!zerocopy) {
      KK_CUDA(cudaMemcpyAsync(s.dev.get(), s.pinned, ch.buf_bytes, cudaMemcpyHostToDevice, rd.stream));
      L.src = s.dev.get();
    }
    L.segs = d_segs + ch.seg_begin;
    L.n_segs = ch.seg_count;
    L.n_tiles = ch.n_tiles;
    L.sched = rd.sched.get<uint32_t>();
    KK_CUDA(launch_convert(L, sm_count, rd.stream));
  });
}

// Stage 1 of a RAW load on local device li: file bytes of its plan part -> local raw image (H2D straight into place) -> peers' raw images
// (COPY launch per chunk, bulk TMA stores over NVLink).
void raw_stage1(kk_model* m, int li, const FdSet& fds) {
  const int part = m->shape.local_parts[(size_t)li];
  const PartPlan& pp = m->plan.parts[(size_t)part];
  if (pp.chunks.empty()) return;
  const int sm_count = m->ctx->devs[(size_t)li].sm_count;
  const DeviceImage& R = m->images[(size_t)li];
  ConvertLaunch base{};
  fill_raw_dsts(m, li, base);
  if (base.n_dst > 0 && !m->shape.multi_proc && !m->shape.peer_ok) fail(KK_EUNSUPPORTED, "KK_FANOUT_RAW needs peer access between the context's devices");
  stream_part(m, li, part, fds, true, [&](Reader& rd, Slot& s, size_t ci) {
    const Chunk& ch = pp.chunks[ci];
    KK_CUDA(cudaMemcpyAsync(R.image.get() + m->img_off[(size_t)part][ci], s.pinned, ch.buf_bytes, cudaMemcpyHostToDevice, rd.stream));
    if (base.n_dst == 0) return;
    ConvertLaunch L = base;
    L.src = R.image.get();
    L.segs = R.copy_segs.get<KKSeg>() + m->chunk_base[(size_t)part] + ci;
    L.n_segs = 1;
    L.n_tiles = (uint32_t)kk_seg_tiles(KK_OP_COPY, align_up(ch.buf_bytes, 16), 0);
    L.sched = rd.sched.get<uint32_t>();
    KK_CUDA(launch_convert(L, sm_count, rd.stream));
  });
}

// Resident staging (untimed): the chunk buffers of plan part `part`, exactly as the streaming path stages them, into `image` at chunk_off.
void stage_image(kk_model* m, int li, int part, const FdSet& fds, uint8_t* image, const std::vector<uint64_t>& chunk_off) {
  const PartPlan& pp = m->plan.parts[(size_t)part];
  stream_part(m, li, part, fds, false, [&](Reader& rd, Slot& s, size_t ci) {
    KK_CUDA(cudaMemcpyAsync(image + chunk_off[ci], s.pinned, pp.chunks[ci].buf_bytes, cudaMemcpyHostToDevice, rd.stream));
  });
}

// Allocate the raw images and build their segment tables: stage 1's copies (one launch per chunk), the fan-out launch's copies and
// stage 2's conversions.
void setup_raw(kk_model* m) {
  const Plan& P = m->plan;
  std::vector<int> all;
  for (int p = 0; p < (int)P.parts.size(); ++p) all.push_back(p);
  const ImageLayout im = lay_out_image(P, all);
  m->img_off = im.chunk_off;
  m->chunk_base.assign(P.parts.size(), 0);
  std::vector<KKSeg> copy_segs;
  std::vector<std::vector<KKSeg>> fanout_segs(P.parts.size());  // [part]: the same copies with tile_begin running over the part
  std::vector<uint32_t> fanout_tiles(P.parts.size(), 0);
  for (size_t p = 0; p < P.parts.size(); ++p) {
    m->chunk_base[p] = (uint32_t)copy_segs.size();
    for (size_t ci = 0; ci < P.parts[p].chunks.size(); ++ci) {
      KKSeg cs{};
      cs.src_off = cs.dst_off = m->img_off[p][ci];
      cs.units = align_up(P.parts[p].chunks[ci].buf_bytes, 16);
      cs.op = KK_OP_COPY;
      copy_segs.push_back(cs);
      cs.tile_begin = fanout_tiles[p];
      fanout_tiles[p] += (uint32_t)kk_seg_tiles(KK_OP_COPY, cs.units, 0);
      fanout_segs[p].push_back(cs);
    }
  }
  m->images.resize(m->pools.size());
  for (size_t li = 0; li < m->images.size(); ++li) {
    const int ordinal = m->ctx->devs[li].ordinal;
    const int part = m->shape.local_parts[li];
    DeviceImage& R = m->images[li];
    // 2 MiB multiples: cheap to map over CUDA IPC (see the slice buffer in model_load)
    R.image = DevBuf(ordinal, align_up(im.bytes ? im.bytes : 256, 2u << 20), "the raw image");
    R.copy_segs = upload_segs(ordinal, copy_segs);
    R.fanout_segs = upload_segs(ordinal, fanout_segs[(size_t)part]);
    R.fanout = {0, (uint32_t)fanout_segs[(size_t)part].size(), fanout_tiles[(size_t)part]};
    R.segs = upload_segs(ordinal, im.segs);
    R.launches = im.launches;
  }
}

// The launches over a device image, each with base's destinations.
std::vector<ConvertLaunch> image_launches(const ConvertLaunch& base, const DeviceImage& im) {
  std::vector<ConvertLaunch> out;
  for (auto& la : im.launches) {
    ConvertLaunch L = base;
    L.src = im.image.get();
    L.segs = im.segs.get<KKSeg>() + la.seg_begin;
    L.n_segs = la.n_segs;
    L.n_tiles = la.n_tiles;
    out.push_back(L);
  }
  return out;
}

// Run launches[li] on the stream of local device li, enqueued on every device before any device is waited for, so that the devices run
// concurrently.  Events bracket the launches alone.  Returns the slowest device's total (ms); per_launch[k] = the slowest k-th launch.
float time_launches(kk_model* m, std::vector<std::vector<ConvertLaunch>>& launches, std::vector<float>* per_launch = nullptr) {
  std::vector<EventSet> evs;
  evs.reserve(launches.size());
  size_t most = 0;
  for (size_t li = 0; li < launches.size(); ++li) {
    Device& dev = m->ctx->devs[li];
    KK_CUDA(cudaSetDevice(dev.ordinal));
    evs.emplace_back(launches[li].size() + 1);
    evs[li].create_all();
    KK_CUDA(cudaEventRecord(evs[li][0], dev.stream));
    for (size_t k = 0; k < launches[li].size(); ++k) {
      launches[li][k].sched = dev.sched.get<uint32_t>();
      KK_CUDA(launch_convert(launches[li][k], dev.sm_count, dev.stream));
      KK_CUDA(cudaEventRecord(evs[li][k + 1], dev.stream));
    }
    most = std::max(most, launches[li].size());
  }
  float worst = 0.f;
  if (per_launch) per_launch->assign(most, 0.f);
  for (size_t li = 0; li < launches.size(); ++li) {
    KK_CUDA(cudaSetDevice(m->ctx->devs[li].ordinal));
    KK_CUDA(cudaStreamSynchronize(m->ctx->devs[li].stream));
    const size_t n = launches[li].size();
    float ms = 0.f;
    KK_CUDA(cudaEventElapsedTime(&ms, evs[li][0], evs[li][n]));
    worst = std::max(worst, ms);
    for (size_t k = 0; per_launch && k < n; ++k) {
      KK_CUDA(cudaEventElapsedTime(&ms, evs[li][k], evs[li][k + 1]));
      (*per_launch)[k] = std::max((*per_launch)[k], ms);
    }
  }
  return worst;
}

// Stage 2: every local device converts the whole gathered image into its own pool.
void convert_local_all(kk_model* m, float* ms_total) {
  std::vector<std::vector<ConvertLaunch>> launches(m->pools.size());
  for (size_t li = 0; li < launches.size(); ++li) {
    ConvertLaunch base{};
    base.n_dst = 1;
    base.flags = format_flags(m);
    base.dst[0] = m->pools[li].ptr;
    launches[li] = image_launches(base, m->images[li]);
  }
  const float ms = time_launches(m, launches);
  if (ms_total) *ms_total = ms;
}

// Stage 2 of a KK_FANOUT_PULL load: one COPY launch whose segments read every attached peer's slice buffer over NVLink (bulk loads)
// and write the local pool.  Segments start with the peer after this rank so that the N ranks do not all read GPU 0 first.
void pull_slices(kk_model* m, float* ms_total) {
  const int n = m->shape.n_parts, me = m->shape.rank;
  const PeerBuf* slice = m->peer[kPeerSlice];
  std::vector<int> peers;
  std::lock_guard<std::mutex> peer_lock(m->peer_mu);
  // Every rank owns a slice buffer (never smaller than 256 B) and every peer's must be attached before stage 2, whether or not the
  // planner gave that rank any bytes: a rank that skipped the exchange is a protocol error of the caller, and reporting success for it
  // only because its part happened to be empty (a checkpoint smaller than one staging chunk) would hide the same mistake at full size.
  for (int k = 1; k < n; ++k) {
    const int r = (me + k) % n;
    if (!slice[r].ptr) fail(KK_ESTATE, "KK_FANOUT_PULL: the slice buffer of rank %d is not attached (kk_peer_attach_buffer, KK_BUF_SLICE)", r);
    if (m->part_range[(size_t)r].second > m->part_range[(size_t)r].first) peers.push_back(r);
  }
  std::vector<std::vector<ConvertLaunch>> launches(1);
  DevBuf table;  // freed after time_launches has waited for the launch that reads it
  if (!peers.empty()) {
    // one src base for the launch: the numerically lowest peer mapping; every segment's src_off is its distance from it
    uintptr_t base = UINTPTR_MAX;
    for (int r : peers) base = std::min(base, (uintptr_t)slice[r].ptr);
    base &= ~(uintptr_t)15;
    std::vector<KKSeg> segs;
    uint64_t tiles = 0;
    for (int r : peers) {
      const uint64_t lo = m->part_range[(size_t)r].first, hi = m->part_range[(size_t)r].second;
      KKSeg sg{};
      sg.src_off = (uint64_t)((uintptr_t)slice[r].ptr - base) + (lo - (lo & ~(uint64_t)255));  // peers allocate from slice_base = lo & ~255
      sg.dst_off = lo;
      sg.units = hi - lo;
      sg.op = KK_OP_COPY;
      sg.tile_begin = (uint32_t)tiles;
      tiles += kk_seg_tiles(KK_OP_COPY, sg.units, 0);
      segs.push_back(sg);
    }
    if (tiles > 0xFFFFFFF0ull) fail(KK_EUNSUPPORTED, "too many tiles for one pull launch");
    table = upload_segs(m->ctx->devs[0].ordinal, segs);
    ConvertLaunch L{};
    L.src = (const uint8_t*)base;
    L.segs = table.get<KKSeg>();
    L.n_segs = (uint32_t)segs.size();
    L.n_tiles = (uint32_t)tiles;
    L.n_dst = 1;
    L.flags = format_flags(m);
    L.dst[0] = m->pools[0].ptr;
    launches[0].push_back(L);
  }
  const float ms = time_launches(m, launches);
  if (ms_total) *ms_total = ms;
}

// RAW, kernel-stage measurement: stage 1's fan-out without the file reads — one COPY launch over all of local device li's own chunks, from
// its raw image into every peer image.
void raw_fanout_launch(kk_model* m, int li, std::vector<ConvertLaunch>& out) {
  ConvertLaunch L{};
  fill_raw_dsts(m, li, L);
  const DeviceImage& R = m->images[(size_t)li];
  if (L.n_dst == 0 || R.fanout.n_segs == 0) return;
  if (R.fanout.n_segs > kMaxSegsPerLaunch) fail(KK_EUNSUPPORTED, "too many chunks for one raw fan-out launch");
  L.src = R.image.get();
  L.segs = R.fanout_segs.get<KKSeg>();
  L.n_segs = R.fanout.n_segs;
  L.n_tiles = R.fanout.n_tiles;
  out.push_back(L);
}

// The merge of m's adapter into every local pool of m, reading the target elements from the same pool of `src`: m itself (kk_load_adapter, in
// place, the load's streams synchronised) or the base m is derived from (kk_derive_adapter, whose op_mu the caller holds).  One launch per
// device over a table of that pool's targets.  Out of place, the bytes outside the targets are copied from src's pool by the copy engines, as
// maximal runs on the device's copy stream, issued on every device before the adapter is read and joined to the merge's stream with an event.
// Everything is enqueued on every device before any device is waited for.  A and B (fp32) and the table live in one buffer per device, freed
// before this returns.
void merge_adapter(kk_model* m, const kk_model* src) {
  const Adapter& A = *m->adapter;
  const size_t nl = m->pools.size();
  std::vector<EventSet> cev;
  cev.reserve(nl);
  for (size_t li = 0; src != m && li < nl; ++li) {
    Device& dev = m->ctx->devs[li];
    const std::vector<Placement>& pl = m->plan.placement_of_part(m->shape.local_parts[li]);
    std::vector<std::pair<uint64_t, uint64_t>> tg;
    for (const LoraPair& p : A.pairs) tg.push_back({pl[p.tensor].pool_offset, pl[p.tensor].pool_offset + pl[p.tensor].nbytes});
    std::sort(tg.begin(), tg.end());
    const uint64_t span = m->pools[li].span();  // src's pool has the same plan bytes and backing, so the same span
    std::vector<std::pair<uint64_t, uint64_t>> runs;  // the complement of the targets in [0, span)
    uint64_t at = 0;
    for (auto& t : tg) {
      if (t.first > at) runs.push_back({at, t.first});
      at = std::max(at, t.second);
    }
    if (at < span) runs.push_back({at, span});
    KK_CUDA(cudaSetDevice(dev.ordinal));
    cev.emplace_back(2);
    cev[li].create_all();
    KK_CUDA(cudaEventRecord(cev[li][0], dev.copy_stream));
    for (auto& r : runs)
      KK_CUDA(cudaMemcpyAsync(m->pools[li].ptr + r.first, src->pools[li].ptr + r.first, r.second - r.first, cudaMemcpyDeviceToDevice, dev.copy_stream));
    KK_CUDA(cudaEventRecord(cev[li][1], dev.copy_stream));
  }
  try {
    double t_host = now_s();
    std::vector<uint64_t> a_off, b_off;
    const std::vector<float> host = read_adapter_f32(A, a_off, b_off);
    t_host = now_s() - t_host;
    std::vector<DevBuf> bufs(nl);
    std::vector<EventSet> evs;
    evs.reserve(nl);
    uint64_t most = 0;
    for (size_t li = 0; li < nl; ++li) {
      Device& dev = m->ctx->devs[li];
      const std::vector<Placement>& pl = m->plan.placement_of_part(m->shape.local_parts[li]);
      std::vector<KKLoraTarget> T;
      uint64_t tiles = 0;
      for (size_t i = 0; i < A.pairs.size(); ++i) {
        const LoraPair& p = A.pairs[i];
        const Placement& q = pl[p.tensor];
        KKLoraTarget t{};
        t.w_off = q.pool_offset;
        t.a_off = a_off[i];
        t.b_off = b_off[i];
        t.rows = (uint32_t)q.shape[0];
        t.cols = (uint32_t)q.shape[1];
        t.row0 = q.slice_dim == 0 ? (uint32_t)q.slice_begin : 0;
        t.col0 = q.slice_dim == 1 ? (uint32_t)q.slice_begin : 0;
        t.a_ld = (uint32_t)p.a.shape[1];
        t.r = p.r;
        t.s = p.s;
        t.out = lora_out_of(q.dtype);
        t.tile_begin = (uint32_t)tiles;
        t.tiles_c = (t.cols + KK_LORA_TILE_C - 1) / KK_LORA_TILE_C;
        const uint32_t n = kk_lora_tiles(t.rows, t.cols);
        if (n == 0) continue;
        tiles += n;
        if (tiles >= (1ull << 31)) fail(KK_EUNSUPPORTED, "adapter: more than 2^31 merge tiles on one device");
        T.push_back(t);
      }
      const uint64_t tb = align_up(T.size() * sizeof(KKLoraTarget), 256), bytes = tb + host.size() * sizeof(float);
      const double tu = now_s();
      KK_CUDA(cudaSetDevice(dev.ordinal));
      bufs[li] = DevBuf(dev.ordinal, bytes, "the adapter");
      if (!T.empty()) KK_CUDA(cudaMemcpy(bufs[li].get(), T.data(), T.size() * sizeof(KKLoraTarget), cudaMemcpyHostToDevice));
      KK_CUDA(cudaMemcpy(bufs[li].get() + tb, host.data(), host.size() * sizeof(float), cudaMemcpyHostToDevice));
      t_host += now_s() - tu;
      evs.emplace_back(2);
      evs[li].create_all();
      KK_CUDA(cudaEventRecord(evs[li][0], dev.stream));
      KK_CUDA(launch_lora_merge(bufs[li].get<KKLoraTarget>(), (uint32_t)T.size(), (uint32_t)tiles, (const float*)(bufs[li].get() + tb),
                                src->pools[li].ptr, m->pools[li].ptr, dev.stream));
      KK_CUDA(cudaEventRecord(evs[li][1], dev.stream));
      if (!cev.empty()) KK_CUDA(cudaStreamWaitEvent(dev.stream, cev[li][1], 0));
      most = std::max(most, bytes);
    }
    float worst = 0.f, worst_copy = 0.f;
    for (size_t li = 0; li < nl; ++li) {
      KK_CUDA(cudaSetDevice(m->ctx->devs[li].ordinal));
      KK_CUDA(cudaStreamSynchronize(m->ctx->devs[li].stream));
      float ms = 0.f;
      KK_CUDA(cudaEventElapsedTime(&ms, evs[li][0], evs[li][1]));
      worst = std::max(worst, ms);
      if (cev.empty()) continue;
      KK_CUDA(cudaEventElapsedTime(&ms, cev[li][0], cev[li][1]));
      worst_copy = std::max(worst_copy, ms);
    }
    m->t_merge = worst / 1e3;
    m->t_copy = worst_copy / 1e3;
    m->t_host = t_host;
    m->adapter_bytes = most;
  } catch (...) {
    // the copies read src's pools and write m's: both must outlive them
    for (size_t li = 0; li < cev.size(); ++li) {
      cudaSetDevice(m->ctx->devs[li].ordinal);
      cudaStreamSynchronize(m->ctx->devs[li].copy_stream);
    }
    throw;
  }
}

// Close the peer buffers this process opened over CUDA IPC and forget every attached one.
void close_peers(kk_model* m) {
  for (auto& kind : m->peer)
    for (PeerBuf& b : kind) {
      if (b.opened_by_ipc) {
        cudaSetDevice(m->ctx->devs[0].ordinal);
        cudaIpcCloseMemHandle(b.ptr);
      }
      b = PeerBuf{};
    }
}

// Peer mappings close first; the model's buffers and pools go with it (the NVLS object after the pools that alias it).
void destroy_model(kk_model* m) {
  close_peers(m);
  delete m;
}

std::string canon(const std::string& p) {
  char buf[4096];
  if (realpath(p.c_str(), buf)) return buf;
  return p;
}

// The registry key of base + adapter: the base model's key and the canonical adapter path.
std::string adapter_key(const std::string& base_key, const std::string& adapter_path) { return base_key + "|a" + canon(adapter_path); }

// The model registered under `key`, refcount + 1, once no load of it is in flight (found = true); or a new model registered there, loading,
// refcount 1, that the caller builds and then publishes or abandons.
kk_model* claim_key(kk_ctx* c, const std::string& key, bool& found) {
  std::unique_lock<std::mutex> lk(c->mu);
  for (;;) {
    auto it = c->models.find(key);
    if (it == c->models.end()) break;
    if (it->second->loading) { c->cv.wait(lk); continue; }
    it->second->refcount++;
    found = true;
    return it->second;
  }
  found = false;
  kk_model* m = new kk_model;
  m->ctx = c;
  m->key = key;
  m->refcount = 1;
  m->loading = true;
  c->models[key] = m;
  return m;
}

void publish(kk_model* m) {
  {
    std::lock_guard<std::mutex> g(m->ctx->mu);
    m->loading = false;
  }
  m->ctx->cv.notify_all();
}

// A claimed model whose build failed: unregistered, waiters woken (they claim the key again), its memory and budget returned.
void abandon(kk_model* m) {
  kk_ctx* c = m->ctx;
  {
    std::lock_guard<std::mutex> g(c->mu);
    c->models.erase(m->key);
  }
  c->cv.notify_all();
  destroy_model(m);
}

// The pools of m's plan and shape on every local device, each reserved on the device's pool budget first (KK_ENOMEM past it), and every
// device's copy of the concatenated segment table.
void alloc_pools(kk_model* m) {
  kk_ctx* c = m->ctx;
  const LoadShape& S = m->shape;
  std::vector<KKSeg> all;
  for (auto& pp : m->plan.parts) all.insert(all.end(), pp.segs.begin(), pp.segs.end());
  const size_t nl = S.local_parts.size();
  m->pools = std::vector<Pool>(nl);
  m->d_segs.resize(nl);
  if (S.order == LoadOrder::kNvls) {
    std::string why;
    if (!plan_allows_multimem(m->plan, &why)) fail(KK_EUNSUPPORTED, "fan-out NVLS: %s", why.c_str());
    std::vector<int> ords;
    for (auto& d : c->devs) ords.push_back(d.ordinal);
    KK_CUDA(cudaSetDevice(ords[0]));  // the driver entry points below want a current context on the calling thread
    m->nvls.reset(new NvlsPools);
    m->nvls->create(ords, m->plan.pool_bytes_of_part(0));
  }
  for (size_t li = 0; li < nl; ++li) {
    Device& d = c->devs[li];
    KK_CUDA(cudaSetDevice(d.ordinal));
    const uint64_t pb = m->plan.pool_bytes_of_part(S.local_parts[li]);
    Pool& pool = m->pools[li];
    {
      std::lock_guard<std::mutex> g(c->mu);
      if (c->cfg.pool_bytes_per_device && d.pool_in_use + pb > c->cfg.pool_bytes_per_device)
        fail(KK_ENOMEM, "device %d: pool budget exceeded (%llu in use + %llu > %llu)", d.ordinal, (unsigned long long)d.pool_in_use,
             (unsigned long long)pb, (unsigned long long)c->cfg.pool_bytes_per_device);
      d.pool_in_use += pb;
      pool.bytes = pb;
      pool.ctx = c;
      pool.dev = &d;
    }
    if (m->nvls) {
      pool.ptr = m->nvls->pool(li);  // already allocated, bound and mapped
    } else if (c->cfg.flags & KK_CFG_VMM_POOLS) {
      // cuMemCreate memory: exported as a POSIX fd (kk_export_fd) that another process maps READ-ONLY, which a cudaIpcMemHandle cannot offer.
      // Mapped read-write here for this device and, in a peer-enabled context, for the other devices (fan-out stores land in it).
      std::vector<int> acc;
      if (c->peer_ok)
        for (auto& dv : c->devs) acc.push_back(dv.ordinal);
      pool.vmm.reset(new VmmAlloc);
      pool.vmm->create(d.ordinal, pb, acc);
      pool.ptr = pool.vmm->ptr();
    } else {
      // whole 2 MiB multiples: the driver sub-allocates smaller requests out of shared 2 MiB blocks, and an IPC handle maps the whole block —
      // a pool that owns its blocks outright cannot expose a neighbouring allocation through its handle (round-1 review)
      pool.mem = DevBuf(d.ordinal, align_up(pb ? pb : 1, 2u << 20), "the pool");
      pool.ptr = pool.mem.get();
    }
    m->d_segs[li] = upload_segs(d.ordinal, all);
  }
}

}  // namespace

Pool::~Pool() {
  mem = DevBuf();  // the memory before its budget: a load that then passes the budget check must find the memory free
  vmm.reset();
  if (!ctx) return;
  std::lock_guard<std::mutex> g(ctx->mu);  // model_load checks the budget under the same lock
  dev->pool_in_use -= bytes;
}

void device_identity(int ordinal, char* bus, size_t bus_cap, char* uuid, size_t uuid_cap) {
  if (bus) {
    KK_CUDA(cudaDeviceGetPCIBusId(bus, (int)bus_cap, ordinal));
    for (char* c = bus; *c; ++c)
      if (*c >= 'A' && *c <= 'F') *c = (char)(*c - 'A' + 'a');
  }
  if (uuid) {
    cudaDeviceProp pr;
    KK_CUDA(cudaGetDeviceProperties(&pr, ordinal));
    const unsigned char* b = (const unsigned char*)pr.uuid.bytes;
    snprintf(uuid, uuid_cap, "GPU-%02x%02x%02x%02x-%02x%02x-%02x%02x-%02x%02x-%02x%02x%02x%02x%02x%02x", b[0], b[1], b[2], b[3], b[4], b[5], b[6], b[7],
             b[8], b[9], b[10], b[11], b[12], b[13], b[14], b[15]);
  }
}

// ---------------------------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------------------------
kk_ctx* ctx_open(const kk_config& cfg_in) {
  kk_config cfg = cfg_in;
  if (cfg.n_devices < 1 || cfg.n_devices > KK_MAX_DEVICES) fail(KK_EINVAL, "n_devices %d out of range 1..%d", cfg.n_devices, KK_MAX_DEVICES);
  for (int i = 0; i < cfg.n_devices; ++i)
    for (int j = 0; j < i; ++j)
      if (cfg.devices[i] == cfg.devices[j]) fail(KK_EINVAL, "device %d listed twice", cfg.devices[i]);
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0)
    fail(KK_ECUDA, "no usable CUDA device (%s); this library has no CPU path", e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
  for (int i = 0; i < cfg.n_devices; ++i)
    if (cfg.devices[i] < 0 || cfg.devices[i] >= count) fail(KK_EINVAL, "device ordinal %d not present (%d devices)", cfg.devices[i], count);
  if (cfg.n_reader_threads == 0) cfg.n_reader_threads = 16;  // 16 x ~4 GB/s of page-cache pread saturates a Gen5 x16 link
  if (cfg.n_staging_buffers == 0) cfg.n_staging_buffers = 2 * cfg.n_reader_threads;
  if (cfg.n_reader_threads > 64) fail(KK_EINVAL, "n_reader_threads %u too large", cfg.n_reader_threads);
  if (cfg.n_staging_buffers < cfg.n_reader_threads) cfg.n_staging_buffers = cfg.n_reader_threads;
  if (cfg.staging_buffer_bytes == 0) cfg.staging_buffer_bytes = 16ull << 20;
  if (cfg.staging_buffer_bytes < (1ull << 20)) fail(KK_EINVAL, "staging_buffer_bytes must be at least 1 MiB");

  std::unique_ptr<kk_ctx> c(new kk_ctx);
  c->cfg = cfg;
  c->slot_bytes = align_up(cfg.staging_buffer_bytes, 2ull << 20);
  c->devs.resize((size_t)cfg.n_devices);
  try {
    // One thread per device, all at once: the pinned ring (cudaHostAlloc pins and maps 0.5 GiB per device by default) dominates kk_open, and eight
    // devices set up one after the other add up to seconds in the one-process shape.  Each
    // thread is bound to its device's NUMA node, so the slots are first-touched / pinned there.
    std::vector<std::exception_ptr> errs((size_t)cfg.n_devices);
    std::vector<std::thread> setup;
    for (int i = 0; i < cfg.n_devices; ++i) {
      c->devs[(size_t)i].ordinal = cfg.devices[i];
      setup.emplace_back([&, i] {
        try {
          Device& d = c->devs[(size_t)i];
          KK_CUDA(cudaSetDevice(d.ordinal));
          cudaDeviceProp prop;
          KK_CUDA(cudaGetDeviceProperties(&prop, d.ordinal));
          // the library carries sm_90a SASS and no PTX: arch-specific code loads on compute capability 9.0 only
          if (prop.major != 9 || prop.minor != 0)
            fail(KK_EUNSUPPORTED, "device %d is sm_%d%d; this build carries sm_90a code only", d.ordinal, prop.major, prop.minor);
          d.sm_count = prop.multiProcessorCount;
          KK_CUDA(kernels_init_device());
          d.kernels_ready = true;
          KK_CUDA(cudaStreamCreateWithFlags(&d.stream, cudaStreamNonBlocking));
          KK_CUDA(cudaStreamCreateWithFlags(&d.copy_stream, cudaStreamNonBlocking));
          d.sched = DevBuf(d.ordinal, 256, "the scheduling words");
          KK_CUDA(cudaMemset(d.sched.get(), 0, 256));
          d.numa_cpus = numa_cpus_of_device(d.ordinal);
          d.readers.resize(cfg.n_reader_threads);
          if (!(cfg.flags & KK_CFG_NO_NUMA_PIN)) pin_this_thread(d.numa_cpus);
          for (uint32_t r = 0; r < cfg.n_reader_threads; ++r) {
            Reader& rd = d.readers[r];
            KK_CUDA(cudaStreamCreateWithFlags(&rd.stream, cudaStreamNonBlocking));
            rd.sched = DevBuf(d.ordinal, 256, "the scheduling words");
            KK_CUDA(cudaMemset(rd.sched.get(), 0, 256));
            uint32_t ns = cfg.n_staging_buffers / cfg.n_reader_threads + (r < cfg.n_staging_buffers % cfg.n_reader_threads ? 1 : 0);
            rd.slots.resize(ns);
            for (auto& s : rd.slots) {
              KK_CUDA(cudaHostAlloc((void**)&s.pinned, c->slot_bytes + 256, cudaHostAllocPortable | cudaHostAllocMapped));
              if (!(cfg.flags & KK_CFG_ZEROCOPY)) s.dev = DevBuf(d.ordinal, c->slot_bytes + 256, "a staging buffer");
              KK_CUDA(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
            }
          }
        } catch (...) {
          errs[(size_t)i] = std::current_exception();
        }
      });
    }
    for (auto& t : setup) t.join();
    for (auto& e : errs)
      if (e) std::rethrow_exception(e);
    if (cfg.flags & KK_CFG_PEER_ALL) {
      for (int i = 0; i < cfg.n_devices; ++i) {
        KK_CUDA(cudaSetDevice(cfg.devices[i]));
        for (int j = 0; j < count; ++j) {
          if (j == cfg.devices[i]) continue;
          int can = 0;
          if (cudaDeviceCanAccessPeer(&can, cfg.devices[i], j) != cudaSuccess || !can) { cudaGetLastError(); continue; }
          cudaError_t pe = cudaDeviceEnablePeerAccess(j, 0);
          if (pe != cudaSuccess) cudaGetLastError();  // already enabled or refused: kk_peer_attach will report a real failure
        }
      }
    }
    c->peer_ok = cfg.n_devices > 1 && !(cfg.flags & KK_CFG_NO_PEER_ACCESS);
    if (c->peer_ok) {
      for (int i = 0; i < cfg.n_devices && c->peer_ok; ++i)
        for (int j = 0; j < cfg.n_devices; ++j) {
          if (i == j) continue;
          int can = 0;
          KK_CUDA(cudaDeviceCanAccessPeer(&can, cfg.devices[i], cfg.devices[j]));
          if (!can) { c->peer_ok = false; break; }
          KK_CUDA(cudaSetDevice(cfg.devices[i]));
          cudaError_t pe = cudaDeviceEnablePeerAccess(cfg.devices[j], 0);
          if (pe == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
          else if (pe != cudaSuccess) { cudaGetLastError(); c->peer_ok = false; break; }
        }
    }
  } catch (...) {
    ctx_close(c.release());
    throw;
  }
  return c.release();
}

void ctx_close(kk_ctx* c) {
  if (!c) return;
  {
    std::lock_guard<std::mutex> g(c->mu);
    if (!c->models.empty()) fail(KK_EBUSY, "%zu model(s) still referenced", c->models.size());
  }
  for (auto& d : c->devs) {
    if (d.ordinal < 0) continue;
    cudaSetDevice(d.ordinal);
    for (auto& rd : d.readers) {
      for (auto& s : rd.slots) {
        if (s.done) cudaEventDestroy(s.done);
        if (s.pinned) cudaFreeHost(s.pinned);
      }
      if (rd.stream) cudaStreamDestroy(rd.stream);
    }
    if (d.stream) cudaStreamDestroy(d.stream);
    if (d.copy_stream) cudaStreamDestroy(d.copy_stream);
  }
  delete c;  // the device buffers go with it
}

// ---------------------------------------------------------------------------------------------
// model
// ---------------------------------------------------------------------------------------------
static void do_load(kk_model* m) {
  const LoadShape& S = m->shape;
  const double t0 = now_s();
  FdSet fds(m->plan.index.shards, map_policy());
  m->t_files_open = now_s() - t0;
  const size_t nl = m->pools.size();
  m->t_part.assign(nl, 0.0);
  ErrorSink sink;
  auto per_dev = [&](int li) {
    try {
      const double a = now_s();
      if (S.order == LoadOrder::kRaw) {
        raw_stage1(m, li, fds);
      } else if (S.every_part) {
        for (int p = 0; p < m->plan.n_parts; ++p) convert_part(m, li, p, fds);
      } else {
        convert_part(m, li, S.local_parts[(size_t)li], fds);
      }
      m->t_part[(size_t)li] = now_s() - a;
    } catch (...) {
      sink.capture();
    }
  };
  std::vector<std::thread> th;
  for (size_t li = 1; li < nl; ++li) th.emplace_back(per_dev, (int)li);
  per_dev(0);
  for (auto& t : th) t.join();
  sink.rethrow();
  if (S.order == LoadOrder::kRaw && !S.two_stage) convert_local_all(m, nullptr);  // one process owns every device: stage 1 is done everywhere
  const double tc = now_s();
  fds.cleanup();  // part of the load: unmapping a checkpoint-sized mapping is not free
  m->t_files_close = now_s() - tc;
  if (m->adapter) merge_adapter(m, m);  // every pool is complete: no load shape that merges has a second stage or a peer's stores still to come
  m->t_load = now_s() - t0;
  m->n_loads++;
  std::lock_guard<std::mutex> g(m->ctx->mu);
  if (!S.two_stage) m->loaded = true;  // a two-stage model is loaded once kk_convert_local has run
}

kk_model* model_load(kk_ctx* c, const std::string& path, const kk_load_opts& opts_in, const std::string& adapter_path) {
  kk_load_opts opts = opts_in;
  if (opts.part_count <= 1) { opts.part_count = 1; opts.part_index = 0; }
  if (!adapter_path.empty()) check_adapter_opts(opts);
  LoadShape shape = resolve_load_shape(opts, c->cfg.n_devices, c->peer_ok);
  if (shape.order == LoadOrder::kNvls) {
    std::vector<int> ords(c->cfg.devices, c->cfg.devices + c->cfg.n_devices);
    std::string why;
    if (!NvlsPools::supported(ords, &why)) fail(KK_EUNSUPPORTED, "fan-out NVLS: this host does not expose it: %s", why.c_str());
  }

  std::ostringstream ks;
  ks << canon(path) << "|m" << opts.mode << "|f" << opts.fanout << "|x" << (opts.flags & ~KK_LOAD_DEFER) << "|p" << opts.part_index << "/" << opts.part_count
     << "|l" << opts.layer_begin << ":" << opts.layer_end;
  const std::string key = adapter_path.empty() ? ks.str() : adapter_key(ks.str(), adapter_path);

  bool found = false;
  kk_model* m = claim_key(c, key, found);
  if (found) return m;
  m->path = path;
  m->opts = opts;
  m->shape = std::move(shape);
  const LoadShape& S = m->shape;
  try {
    double t0 = now_s();
    Index ix = index_for_load(path, opts.flags, opts.layer_begin, opts.layer_end);
    m->t_index = now_s() - t0;
    t0 = now_s();
    m->plan = build_plan(std::move(ix), opts.mode, opts.flags & ~KK_LOAD_DEFER, S.n_parts, c->slot_bytes);
    if (!adapter_path.empty()) m->adapter.reset(new Adapter(match_adapter(adapter_path, path, opts.flags, m->plan)));
    m->t_plan = now_s() - t0;
    t0 = now_s();
    alloc_pools(m);
    if (S.order == LoadOrder::kRaw) setup_raw(m);
    if (S.order == LoadOrder::kPull) {
      m->part_range.assign((size_t)m->plan.n_parts, {0, 0});
      for (int p = 0; p < m->plan.n_parts; ++p)
        if (!part_pool_range(m->plan, p, m->part_range[(size_t)p].first, m->part_range[(size_t)p].second))
          fail(KK_EUNSUPPORTED, "KK_FANOUT_PULL cannot be combined with transposing loads (their output is not one contiguous pool range per rank)");
      const auto& mine = m->part_range[(size_t)S.rank];
      m->slice_base = mine.first & ~(uint64_t)255;
      const uint64_t sb = mine.second > m->slice_base ? mine.second - m->slice_base : 0;
      // whole 2 MiB multiples, like the pools: cudaIpcOpenMemHandle of such an allocation is far cheaper than of one the driver carved out of
      // shared blocks (at N = 8, seven rounded 16 GB pools map faster than seven 2 GB slice buffers of odd size)
      m->slice_buf = DevBuf(c->devs[0].ordinal, align_up(sb ? sb : 256, 2u << 20), "the slice buffer");
    }
    m->t_alloc = now_s() - t0;
    if (!(opts.flags & KK_LOAD_DEFER)) {
      do_load(m);
      if (S.order == LoadOrder::kRaw && !S.two_stage) m->images.clear();  // the gathered file bytes are not needed once the pools are built
    }
  } catch (...) {
    abandon(m);
    throw;
  }
  publish(m);
  return m;
}

kk_model* derive_model(kk_model* base, const std::string& adapter_path) {
  kk_ctx* c = base->ctx;
  check_adapter_opts(base->opts);  // before the state check: a load shape that cannot merge never will
  {
    std::lock_guard<std::mutex> g(c->mu);
    if (base->adapter) fail(KK_EINVAL, "kk_derive_adapter: the base model carries an adapter already (adapters do not stack)");
    if (!base->loaded) fail(KK_ESTATE, "kk_derive_adapter: the base model is not loaded (kk_load_part / kk_convert_local first)");
  }
  const double t0 = now_s();
  bool found = false;
  kk_model* m = claim_key(c, adapter_key(base->key, adapter_path), found);
  if (found) return m;
  try {
    // the base's path, options, plan and shape never change once it is published
    m->path = base->path;
    m->opts = base->opts;
    m->shape = base->shape;
    m->plan = base->plan;
    m->base_key = base->key;
    m->adapter.reset(new Adapter(match_adapter(adapter_path, m->path, m->opts.flags, m->plan)));
    m->t_plan = now_s() - t0;
    const double ta = now_s();
    alloc_pools(m);
    // a deferred RAW model keeps its raw image for kk_load_part, as the load of base + adapter does; other shapes that merge have none
    if (m->shape.order == LoadOrder::kRaw && (m->opts.flags & KK_LOAD_DEFER)) setup_raw(m);
    m->t_alloc = now_s() - ta;
    {
      std::lock_guard<std::mutex> op(base->op_mu);  // a kk_load_part of the base must not rewrite its pools under the copy
      merge_adapter(m, base);
    }
    std::lock_guard<std::mutex> g(c->mu);
    m->loaded = true;
  } catch (...) {
    abandon(m);
    throw;
  }
  publish(m);
  return m;
}

void model_load_part(kk_model* m) {
  std::lock_guard<std::mutex> op(m->op_mu);
  if (m->shape.order == LoadOrder::kRaw && m->images.empty()) fail(KK_ESTATE, "the raw image of this model has been released");
  do_load(m);
}

void model_convert_local(kk_model* m, float* ms_total) {
  std::lock_guard<std::mutex> op(m->op_mu);
  if (m->shape.order == LoadOrder::kPull) pull_slices(m, ms_total);
  else if (m->shape.order == LoadOrder::kRaw && !m->images.empty()) convert_local_all(m, ms_total);
  else fail(KK_ESTATE, "kk_convert_local only applies to KK_FANOUT_RAW models with a live raw image and to KK_FANOUT_PULL models");
  std::lock_guard<std::mutex> g(m->ctx->mu);
  m->loaded = true;
}

void model_export_raw(kk_model* m, int li, void* handle_out) {
  if (m->shape.order != LoadOrder::kRaw || m->images.empty()) fail(KK_ESTATE, "this model has no raw image");
  KK_CUDA(cudaSetDevice(m->ctx->devs[(size_t)li].ordinal));
  cudaIpcMemHandle_t h;
  KK_CUDA(cudaIpcGetMemHandle(&h, m->images[(size_t)li].image.get()));
  memcpy(handle_out, &h, sizeof h);
}

void model_export_slice(kk_model* m, void* handle_out, bool as_pointer) {
  if (m->shape.order != LoadOrder::kPull || !m->slice_buf) fail(KK_ESTATE, "this model has no slice buffer (KK_FANOUT_PULL only)");
  if (as_pointer) {
    void* p = m->slice_buf.get();
    memcpy(handle_out, &p, sizeof p);
    return;
  }
  KK_CUDA(cudaSetDevice(m->ctx->devs[0].ordinal));
  cudaIpcMemHandle_t h;
  KK_CUDA(cudaIpcGetMemHandle(&h, m->slice_buf.get()));
  memcpy(handle_out, &h, sizeof h);
}

// NVLink probe (measurement only): copy-engine read of `nbytes` from the attached buffer of rank `rank` (its pool, or its slice buffer
// in a PULL load) into a local scratch, one untimed pass first, CUDA events on the device's stream.  Run by every rank at once against
// its ring neighbour this is the per-GPU ingress rate the fan-out's roofline is quoted against — measured in the run, not assumed.
void model_probe_peer(kk_model* m, int rank, PeerKind kind, uint64_t& nbytes, float* ms) {
  std::lock_guard<std::mutex> op(m->op_mu);
  if (rank < 0 || rank >= KK_MAX_DEVICES) fail(KK_EINVAL, "bad peer rank %d", rank);
  uint64_t avail = 0;
  if (kind == kPeerPool) {
    avail = m->pools.empty() ? 0 : m->pools[0].bytes;
  } else if (kind == kPeerRaw) {
    avail = m->images.empty() ? 0 : m->images[0].image.bytes();
  } else if ((size_t)rank < m->part_range.size()) {
    const auto& pr = m->part_range[(size_t)rank];
    avail = pr.second > (pr.first & ~(uint64_t)255) ? pr.second - (pr.first & ~(uint64_t)255) : 0;
  }
  const uint8_t* src;
  {
    std::lock_guard<std::mutex> g(m->peer_mu);
    src = (const uint8_t*)m->peer[kind][rank].ptr;
  }
  if (!src) fail(KK_ESTATE, "probe: rank %d has no attached buffer of that kind", rank);
  nbytes = std::min(nbytes, avail) & ~(uint64_t)255;
  if (!nbytes) fail(KK_EINVAL, "probe: nothing to copy from rank %d", rank);
  Device& dev = m->ctx->devs[0];
  DevBuf tmp(dev.ordinal, nbytes, "the peer probe");
  EventSet ev(2);
  ev.create_all();
  KK_CUDA(cudaMemcpyAsync(tmp.get(), src, nbytes, cudaMemcpyDeviceToDevice, dev.stream));
  KK_CUDA(cudaEventRecord(ev[0], dev.stream));
  KK_CUDA(cudaMemcpyAsync(tmp.get(), src, nbytes, cudaMemcpyDeviceToDevice, dev.stream));
  KK_CUDA(cudaEventRecord(ev[1], dev.stream));
  KK_CUDA(cudaStreamSynchronize(dev.stream));
  KK_CUDA(cudaEventElapsedTime(ms, ev[0], ev[1]));
  if (*ms < 0.f) *ms = 0.f;
}

void model_release(kk_model* m) {
  kk_ctx* c = m->ctx;
  {
    std::lock_guard<std::mutex> g(c->mu);
    if (m->refcount <= 0) fail(KK_ESTATE, "release of a model with refcount %d", m->refcount);
    if (--m->refcount > 0) return;
    c->models.erase(m->key);
  }
  destroy_model(m);
}

void model_peer_attach(kk_model* m, PeerKind kind, int rank, const void* handle, bool is_ipc) {
  // Pool and raw tables are read by a running load: those attach under op_mu.  Slice buffers do not: stage 1 of a PULL load (kk_load_part)
  // writes only this rank's own pool and slice buffer, so the caller may map the peers' slice buffers on another thread while it runs.
  // The mapping itself happens outside peer_mu (it is the slow part; several ranks may be attached concurrently), only the table update is locked.
  std::unique_lock<std::mutex> op(m->op_mu, std::defer_lock);
  if (kind != kPeerSlice) op.lock();
  const LoadShape& S = m->shape;
  if (kind == kPeerRaw && S.order != LoadOrder::kRaw) fail(KK_ESTATE, "raw peer attach needs a KK_FANOUT_RAW model");
  if (kind == kPeerSlice && S.order != LoadOrder::kPull) fail(KK_ESTATE, "slice attach needs a KK_FANOUT_PULL model");
  if (!S.multi_proc) fail(KK_ESTATE, "peer attach needs a multi-process (part_count > 1) model");
  if (rank < 0 || rank >= S.n_parts || rank == S.rank) fail(KK_EINVAL, "bad peer rank %d", rank);
  // a multi-process SCATTER model with KK_LOAD_SCATTER_EXCHANGE is the one that has an xdst table
  if (kind == kPeerPool && m->plan.mode != KK_MODE_BROADCAST && !S.xdst)
    fail(KK_ESTATE, "peer attach only applies to BROADCAST models and to SCATTER models loaded with KK_LOAD_SCATTER_EXCHANGE");
  PeerBuf& b = m->peer[kind][rank];
  {
    std::lock_guard<std::mutex> g(m->peer_mu);
    if (b.ptr) fail(KK_ESTATE, "peer rank %d already attached", rank);
  }
  KK_CUDA(cudaSetDevice(m->ctx->devs[0].ordinal));
  void* p = nullptr;
  if (is_ipc) {
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof h);
    KK_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  } else {
    memcpy(&p, handle, sizeof p);
    if (!p) fail(KK_EINVAL, "null device pointer");
  }
  std::lock_guard<std::mutex> g(m->peer_mu);
  if (b.ptr) {  // lost a race against a concurrent slice attach of the same rank
    if (is_ipc) cudaIpcCloseMemHandle(p);
    fail(KK_ESTATE, "peer rank %d already attached", rank);
  }
  b.ptr = p;
  b.opened_by_ipc = is_ipc;
}

void model_peer_detach_all(kk_model* m) {
  std::lock_guard<std::mutex> op(m->op_mu);  // the destination tables are read by a running load
  std::lock_guard<std::mutex> pg(m->peer_mu);
  close_peers(m);
}

int model_local_device(kk_model* m, int ordinal) {
  for (size_t li = 0; li < m->pools.size(); ++li)
    if (m->ctx->devs[li].ordinal == ordinal) return (int)li;
  fail(KK_EINVAL, "device %d holds no pool of this model", ordinal);
}

void model_pool_ipc_handle(kk_model* m, int li, void* handle_out) {
  std::lock_guard<std::mutex> g(m->export_mu);
  if (m->pool_handle_cache.size() < m->pools.size()) m->pool_handle_cache.resize(m->pools.size());
  auto& c = m->pool_handle_cache[(size_t)li];
  if (c.empty()) {
    KK_CUDA(cudaSetDevice(m->ctx->devs[(size_t)li].ordinal));
    cudaIpcMemHandle_t h;
    KK_CUDA(cudaIpcGetMemHandle(&h, m->pools[(size_t)li].ptr));
    static_assert(sizeof h == KK_IPC_HANDLE_BYTES, "ipc handle size");
    c.assign((const uint8_t*)&h, (const uint8_t*)&h + sizeof h);
  }
  memcpy(handle_out, c.data(), c.size());
}

static std::string build_manifest(kk_model* m, int li);
std::string model_manifest(kk_model* m, int li) {
  std::lock_guard<std::mutex> g(m->export_mu);
  if (m->manifest_cache.size() < m->pools.size()) m->manifest_cache.resize(m->pools.size());
  auto& c = m->manifest_cache[(size_t)li];
  if (c.empty()) c = build_manifest(m, li);
  return c;
}

static std::string build_manifest(kk_model* m, int li) {
  const auto& pl = m->plan.placement_of_part(m->shape.local_parts[(size_t)li]);
  const auto& T = m->plan.index.tensors;
  std::ostringstream o;
  // "device" is the ordinal in THIS process (diagnostics only); a consumer in another process or container finds the GPU by its UUID / PCI bus id
  const int ordinal = m->ctx->devs[(size_t)li].ordinal;
  char bus[32] = "", uuid[48] = "";
  try {
    device_identity(ordinal, bus, sizeof bus, uuid, sizeof uuid);
  } catch (const Error&) {  // the manifest says "unknown" with empty strings
    cudaGetLastError();
    bus[0] = uuid[0] = 0;
  }
  o << "{\"apiVersion\":\"kukeon.gpupool/v1\",\"kind\":\"PoolManifest\",\"device\":" << ordinal << ",\"deviceUUID\":\"" << uuid << "\",\"pciBusId\":\"" << bus
    << "\",\"poolBytes\":" << m->pools[(size_t)li].bytes << ",\"mode\":" << m->plan.mode << ",\"format\":\"" << m->plan.index.format
    << "\",\"align\":" << KK_POOL_ALIGN;
  const Index& ix = m->plan.index;
  if (!ix.hf_arch.empty()) o << ",\"layout\":\"hf\",\"architecture\":\"" << json_escape(ix.hf_arch) << "\"";
  if (ix.layer_end) o << ",\"layerBegin\":" << ix.layer_begin << ",\"layerEnd\":" << ix.layer_end << ",\"nLayers\":" << ix.n_layers;
  if (m->adapter) o << ",\"adapter\":{\"path\":\"" << json_escape(m->adapter->path) << "\",\"nTensors\":" << m->adapter->pairs.size() << "}";
  o << ",\"tensors\":[";
  for (size_t i = 0; i < T.size(); ++i) {
    const DtypeInfo* di = dtype_info(pl[i].dtype);
    if (i) o << ",";
    o << "{\"name\":\"" << json_escape(T[i].name) << "\",\"dtype\":\"" << (di ? di->name : "?") << "\",\"shape\":[";
    for (size_t d = 0; d < pl[i].shape.size(); ++d) o << (d ? "," : "") << pl[i].shape[d];
    o << "],\"offset\":" << pl[i].pool_offset << ",\"nbytes\":" << pl[i].nbytes;
    if (pl[i].slice_dim != kNoSlice) o << ",\"sliceDim\":" << pl[i].slice_dim << ",\"sliceBegin\":" << pl[i].slice_begin;
    o << "}";
  }
  o << "]}";
  return o.str();
}

std::string model_stats(kk_model* m) {
  std::ostringstream o;
  o.precision(9);
  const std::vector<int>& local_parts = m->shape.local_parts;
  uint64_t src = 0, out = 0;
  for (size_t li = 0; li < local_parts.size(); ++li) {
    const PartPlan& pp = m->plan.parts[(size_t)local_parts[li]];
    src += pp.src_bytes;
    out += pp.out_bytes;
  }
  o << "{\"n_tensors\":" << m->plan.index.tensors.size() << ",\"n_shards\":" << m->plan.index.shards.size()
    << ",\"file_bytes\":" << m->plan.file_bytes << ",\"pool_bytes\":" << m->plan.pool_bytes_of_part(local_parts[0])
    << ",\"n_parts\":" << m->plan.n_parts << ",\"local_src_bytes\":" << src << ",\"local_out_bytes\":" << out
    << ",\"index_s\":" << m->t_index << ",\"plan_s\":" << m->t_plan << ",\"alloc_s\":" << m->t_alloc << ",\"load_s\":" << m->t_load
    << ",\"n_loads\":" << m->n_loads << ",\"readers\":{\"threads\":" << m->rd_threads << ",\"slot_wait_s\":" << m->rd_wait_ns.load() / 1e9 << ",\"pread_s\":" << m->rd_pread_ns.load() / 1e9
    << ",\"issue_s\":" << m->rd_issue_ns.load() / 1e9 << ",\"drain_s\":" << m->rd_drain_ns.load() / 1e9 << ",\"files_open_s\":" << m->t_files_open << ",\"files_close_s\":" << m->t_files_close << "},\"load_gbps\":" << (m->t_load > 0 ? (double)src / m->t_load / 1e9 : 0.0) << ",\"parts\":[";
  for (size_t li = 0; li < local_parts.size(); ++li) {
    const int part = local_parts[li];
    const PartPlan& pp = m->plan.parts[(size_t)part];
    uint64_t lo, hi;
    part_pool_range(m->plan, part, lo, hi);
    uint64_t tiles = 0;
    for (auto& ch : pp.chunks) tiles += ch.n_tiles;
    if (li) o << ",";
    o << "{\"part\":" << part << ",\"device\":" << m->ctx->devs[li].ordinal << ",\"chunks\":" << pp.chunks.size()
      << ",\"segs\":" << pp.segs.size() << ",\"tiles\":" << tiles << ",\"src_bytes\":" << pp.src_bytes << ",\"out_bytes\":" << pp.out_bytes
      << ",\"pool_lo\":" << lo << ",\"pool_hi\":" << hi << ",\"seconds\":" << (li < m->t_part.size() ? m->t_part[li] : 0.0) << "}";
  }
  o << "]";
  if (m->adapter)
    o << ",\"adapter\":{\"path\":\"" << json_escape(m->adapter->path) << "\",\"n_tensors\":" << m->adapter->pairs.size()
      << ",\"n_skipped\":" << m->adapter->skipped.size() << ",\"bytes\":" << m->adapter_bytes << ",\"t_merge\":" << m->t_merge << "}";
  if (!m->base_key.empty())
    o << ",\"derive\":{\"base_key\":\"" << json_escape(m->base_key) << "\",\"t_copy\":" << m->t_copy << ",\"t_merge\":" << m->t_merge
      << ",\"t_host\":" << m->t_host << "}";
  o << "}";
  return o.str();
}

// ---------------------------------------------------------------------------------------------
// resident image: kernel-stage measurement with the source bytes already in HBM
// ---------------------------------------------------------------------------------------------
void model_stage_resident(kk_model* m) {
  std::lock_guard<std::mutex> op(m->op_mu);
  const bool raw = m->shape.order == LoadOrder::kRaw;
  const std::vector<int>& local_parts = m->shape.local_parts;
  if (!raw) m->images.clear();
  else if (m->images.empty()) fail(KK_ESTATE, "the raw image of this model has been released");
  FdSet fds(m->plan.index.shards, map_policy());
  if (raw) {  // RAW: the resident image IS the raw image; stage this process's own part(s), no fan-out
    for (size_t li = 0; li < local_parts.size(); ++li)
      stage_image(m, (int)li, local_parts[li], fds, m->images[li].image.get(), m->img_off[(size_t)local_parts[li]]);
    return;
  }
  std::vector<DeviceImage> images(local_parts.size());
  for (size_t li = 0; li < local_parts.size(); ++li) {
    const int ordinal = m->ctx->devs[li].ordinal;
    const ImageLayout im = lay_out_image(m->plan, {local_parts[li]});
    DeviceImage& R = images[li];
    R.image = DevBuf(ordinal, im.bytes ? im.bytes : 256, "the resident image");
    stage_image(m, (int)li, local_parts[li], fds, R.image.get(), im.chunk_off[0]);
    R.segs = upload_segs(ordinal, im.segs);
    R.launches = im.launches;
  }
  m->images = std::move(images);
}

void model_unstage_resident(kk_model* m) {
  std::lock_guard<std::mutex> op(m->op_mu);
  if (m->shape.order == LoadOrder::kRaw) return;  // the raw image lives as long as a deferred RAW model does
  m->images.clear();
}

// RAW: the stage-1 fan-out alone (own part of the image -> every peer image), one launch per local device.  Otherwise the resident image's
// launches on every local device.
void model_convert_resident(kk_model* m, float* ms_total, float* ms_per_launch, size_t cap, size_t* n_launches) {
  std::lock_guard<std::mutex> op(m->op_mu);
  const size_t nl = m->pools.size();
  std::vector<std::vector<ConvertLaunch>> launches(nl);
  if (m->shape.order == LoadOrder::kRaw) {
    if (m->images.empty()) fail(KK_ESTATE, "the raw image of this model has been released");
    for (size_t li = 0; li < nl; ++li) raw_fanout_launch(m, (int)li, launches[li]);
  } else {
    if (m->images.size() != nl) fail(KK_ESTATE, "kk_stage_resident has not been called");
    for (size_t li = 0; li < nl; ++li) {
      ConvertLaunch base{};
      fill_dsts(m, (int)li, base);
      launches[li] = image_launches(base, m->images[li]);
    }
  }
  std::vector<float> per;
  const float ms = time_launches(m, launches, &per);
  if (ms_total) *ms_total = ms;
  if (n_launches) *n_launches = per.size();
  if (ms_per_launch)
    for (size_t k = 0; k < per.size() && k < cap; ++k) ms_per_launch[k] = per[k];
}

}  // namespace kk
