// Context (daemon-lifetime GPU pool manager) and model (one resident checkpoint) objects behind the C ABI.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <condition_variable>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "kk_common.hpp"
#include "kk_kernels.cuh"
#include "kk_nvls.hpp"
#include "kk_plan.hpp"
#include "kk_vmm.hpp"

namespace kk {

#define KK_CUDA(expr)                                                                               \
  do {                                                                                              \
    cudaError_t _e = (expr);                                                                        \
    if (_e != cudaSuccess) ::kk::fail(KK_ECUDA, "%s: %s (%s)", #expr, cudaGetErrorString(_e), cudaGetErrorName(_e)); \
  } while (0)

struct Slot {
  uint8_t* pinned = nullptr;  // cudaHostAlloc'd, also mapped into the device address space
  uint8_t* dev = nullptr;     // device staging buffer of the same size
  cudaEvent_t done = nullptr; // recorded after the convert kernel that consumed this slot
};

struct Reader {
  cudaStream_t stream = nullptr;
  uint32_t* sched = nullptr;  // two zeroed device words: the tile-scheduling counters of the launches on `stream` (ConvertLaunch::sched)
  std::vector<Slot> slots;
};

struct Device {
  // One staging pipeline at a time per device: the reader slots and streams below belong to whichever load holds this.
  // (Concurrent loads of different checkpoints on one GPU serialise here; its PCIe link is the bottleneck anyway.)
  std::unique_ptr<std::mutex> load_mu{new std::mutex};
  int ordinal = -1;
  int sm_count = 0;
  std::vector<Reader> readers;
  cudaStream_t stream = nullptr;  // resident launches, checksum, misc
  uint32_t* sched = nullptr;      // tile-scheduling counters of the launches on `stream` (first 8 of 256 zeroed bytes)
  std::unique_ptr<std::mutex> sum_mu{new std::mutex};  // kk_checksum's accumulator is the 8 bytes at sched + 32 words: no cudaMalloc / cudaFree per call
  uint64_t pool_in_use = 0;
  bool kernels_ready = false;
  std::vector<int> numa_cpus;  // CPUs local to the device's PCIe root (reader threads are pinned there)
};

// Peer buffers of a multi-process model, attached by rank: the other ranks' pools (fan-out destinations), raw images (KK_FANOUT_RAW
// stage 1) and slice buffers (KK_FANOUT_PULL stage 2).
enum PeerKind { kPeerPool = 0, kPeerRaw, kPeerSlice, kPeerKinds };
struct PeerBuf {
  void* ptr = nullptr;
  bool opened_by_ipc = false;  // false: a caller-owned device pointer (KK_BUF_*_PTR), never closed by us
};

// One convert launch over a device image: its slice of the image's rebased segment table.
struct ImageLaunch {
  uint32_t seg_begin, n_segs, n_tiles;
};

}  // namespace kk

struct kk_ctx {
  kk_config cfg{};
  uint64_t slot_bytes = 0;
  std::vector<kk::Device> devs;
  bool peer_ok = false;  // every device pair has peer access enabled
  std::mutex mu;
  std::condition_variable cv;
  std::map<std::string, kk_model*> models;
};

struct kk_model {
  kk_ctx* ctx = nullptr;
  std::string key;
  kk::Plan plan;
  kk_load_opts opts{};
  // local devices that hold a pool, as indices into ctx->devs; local_parts[i] is the plan part device i ingests
  std::vector<int> dev_idx;
  std::vector<int> local_parts;
  std::vector<uint8_t*> pools;       // per local device
  std::vector<uint64_t> pool_bytes;  // per local device
  // What kk_export hands out is fixed once the pools exist: the manifest text and the pool's CUDA IPC handle are built on first use and kept.  Every
  // cell that mounts the model exports again, and the calls underneath (cudaIpcGetMemHandle, cudaGetDeviceProperties) go through the driver's
  // system-wide lock, where they wait behind whatever another process on the host is doing in the driver.
  std::mutex export_mu;
  std::vector<std::string> manifest_cache;               // per local device, empty = not built yet
  std::vector<std::vector<uint8_t>> pool_handle_cache;   // per local device, empty = not asked yet
  std::vector<KKSeg*> d_segs;        // per local device: device copy of its part's segment table
  kk::PeerBuf peer[kk::kPeerKinds][KK_MAX_DEVICES];  // [kind][rank]
  // resident image (kernel-stage measurement)
  struct Resident {
    uint8_t* image = nullptr;
    KKSeg* d_segs = nullptr;
    std::vector<kk::ImageLaunch> launches;
  };
  std::vector<Resident> resident;  // per local device
  // KK_FANOUT_RAW: the file bytes of every part are all-gathered into a per-device raw image (stage 1, fan-out of
  // the *quantised* bytes), then every device converts the whole image into its own pool (stage 2).
  struct Raw {
    uint8_t* image = nullptr;
    uint64_t bytes = 0;
    KKSeg* d_copy_segs = nullptr;  // one COPY segment per chunk of every part: [chunk_base[part] + ci]
    KKSeg* d_conv_segs = nullptr;  // every part's segments rebased onto the image
    std::vector<kk::ImageLaunch> conv_launches;
  };
  std::vector<Raw> raw;                         // per local device (empty unless fanout == RAW)
  std::vector<std::vector<uint64_t>> img_off;   // [part][chunk] offset of the chunk buffer inside the raw image
  std::vector<uint32_t> chunk_base;             // prefix sum of chunk counts per part
  // KK_FANOUT_PULL (one process per GPU): this rank's part of the pool, [slice_lo, slice_hi), also lives in slice_buf (a separate,
  // small allocation — the only thing peers have to map); slice_buf[0] corresponds to pool offset slice_base
  uint8_t* slice_buf = nullptr;
  uint64_t slice_base = 0;
  std::vector<std::pair<uint64_t, uint64_t>> part_range;  // [lo, hi) pool bytes every part produces
  bool raw_staged = false;                      // stage 1 complete on this process since the last conversion
  // KK_FANOUT_NVLS (one process, >= 2 devices): the pools are VMM allocations bound to one multicast object; pools[i] then
  // aliases nvls->pool(i) and must not be cudaFree'd
  std::unique_ptr<kk::NvlsPools> nvls;
  // KK_CFG_VMM_POOLS: pools[i] aliases vmm[i]->ptr() (cuMemCreate memory, exportable as a POSIX fd and mappable read-only elsewhere); never cudaFree'd
  std::vector<std::unique_ptr<kk::VmmAlloc>> vmm;
  // state
  std::mutex op_mu;  // serialises the data-moving calls on ONE model (kk_load_part, kk_convert_local, kk_*_resident) against each other
  std::mutex peer_mu;  // guards peer[]; slice attach takes only this lock: stage 1 of a PULL load never reads the slice table, so slice buffers may be attached WHILE kk_load_part runs
                       // (cudaIpcOpenMemHandle is the expensive part of time-to-ready in the one-process-per-GPU shape); lock order op_mu -> peer_mu
  int refcount = 0;
  bool loading = true;
  bool loaded = false;
  int load_error = 0;
  std::string load_error_msg;
  // stats
  double t_index = 0, t_plan = 0, t_alloc = 0, t_load = 0;
  uint64_t n_loads = 0;
  std::vector<double> t_part;  // per local device wall seconds of the last load
  // where the reader threads of the last kk_load_part spent their time, summed over threads (seconds): waiting for a free slot (= for the GPU
  // to finish the chunk that used it), in pread, issuing the H2D copy + launch, and in the final stream synchronise; plus the thread count
  std::atomic<uint64_t> rd_wait_ns{0}, rd_pread_ns{0}, rd_issue_ns{0}, rd_drain_ns{0};
  double t_files_open = 0, t_files_close = 0;  // of the last load: open + map, unmap + close
  uint32_t rd_threads = 0;
};

namespace kk {

kk_ctx* ctx_open(const kk_config& cfg);
void ctx_close(kk_ctx* c);

kk_model* model_load(kk_ctx* c, const std::string& path, const kk_load_opts& opts);
void model_load_part(kk_model* m);
void model_release(kk_model* m);
void model_peer_attach(kk_model* m, PeerKind kind, int rank, const void* handle, bool is_ipc);
void model_export_raw(kk_model* m, int local, void* handle_out);
void model_export_slice(kk_model* m, void* handle_out, bool as_pointer);
void model_convert_local(kk_model* m, float* ms_total);
void model_probe_peer(kk_model* m, int rank, PeerKind kind, uint64_t& nbytes, float* ms);
void model_peer_detach_all(kk_model* m);
int model_local_device(kk_model* m, int ordinal);  // index into m->dev_idx or throws
std::string model_manifest(kk_model* m, int local);
void model_pool_ipc_handle(kk_model* m, int local, void* handle_64B);  // cudaIpcGetMemHandle of the pool, once per model and device
std::string model_stats(kk_model* m);
void model_stage_resident(kk_model* m);
void model_unstage_resident(kk_model* m);
void model_convert_resident(kk_model* m, float* ms_total, float* ms_per_launch, size_t cap, size_t* n_launches);

}  // namespace kk
