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
#include "kk_mem.hpp"
#include "kk_plan.hpp"

namespace kk {

// CUDA events that must not leak when a KK_CUDA check throws half way through a function.
struct EventSet {
  std::vector<cudaEvent_t> ev;
  explicit EventSet(size_t n = 0) : ev(n, nullptr) {}
  cudaEvent_t& operator[](size_t i) { return ev[i]; }
  size_t size() const { return ev.size(); }
  void create_all() {
    for (auto& e : ev) KK_CUDA(cudaEventCreate(&e));
  }
  ~EventSet() {
    for (auto e : ev)
      if (e) cudaEventDestroy(e);
  }
  EventSet(const EventSet&) = delete;
  EventSet& operator=(const EventSet&) = delete;
  EventSet(EventSet&& o) noexcept : ev(std::move(o.ev)) { o.ev.clear(); }
};

// PCI bus id (lower case, as /proc/driver/nvidia/gpus/ names it) and UUID ("GPU-…") of a CUDA device; a null output is skipped.  Throws KK_ECUDA.
void device_identity(int ordinal, char* bus, size_t bus_cap, char* uuid, size_t uuid_cap);

struct Slot {
  uint8_t* pinned = nullptr;  // cudaHostAlloc'd, also mapped into the device address space
  DevBuf dev;                 // device staging buffer of the same size
  cudaEvent_t done = nullptr; // recorded after the convert kernel that consumed this slot
};

struct Reader {
  cudaStream_t stream = nullptr;
  DevBuf sched;  // two zeroed device words: the tile-scheduling counters every launch on `stream` needs (ConvertLaunch::sched)
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
  DevBuf sched;                   // tile-scheduling counters every launch on `stream` needs (first 8 of 256 zeroed bytes)
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

// Chunk buffers of plan parts staged back to back in HBM (lay_out_image): the resident image of kk_stage_resident, and the raw image of a
// KK_FANOUT_RAW load, into which the file bytes of every part are all-gathered (stage 1) before every device converts all of it (stage 2).
struct DeviceImage {
  DevBuf image;
  DevBuf segs;      // every part's segments rebased onto the image
  std::vector<ImageLaunch> launches;
  DevBuf copy_segs;  // RAW: one COPY segment per chunk of every part, [kk_model::chunk_base[part] + ci]
  DevBuf fanout_segs;  // RAW: the same for this device's own part, tile_begin running, as the one launch `fanout`
  ImageLaunch fanout{};
};

// The pool of one local device: cudaMalloc memory in whole 2 MiB multiples, a VMM allocation, or an alias into kk_model::nvls.  Its plan
// bytes are reserved on Device::pool_in_use, and returned under kk_ctx::mu once the memory is gone.
struct Pool {
  uint8_t* ptr = nullptr;
  uint64_t bytes = 0;             // plan bytes
  DevBuf mem;                     // cudaMalloc backing
  std::unique_ptr<VmmAlloc> vmm;  // KK_CFG_VMM_POOLS backing
  kk_ctx* ctx = nullptr;          // set once `bytes` are reserved on dev->pool_in_use
  Device* dev = nullptr;
  bool is_nvls() const { return ptr && !mem && !vmm; }
  Pool() = default;
  Pool(const Pool&) = delete;
  ~Pool();
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
  kk::LoadShape shape;  // local device li (every per-device vector below) is ctx->devs[li]
  // KK_FANOUT_NVLS (one process, >= 2 devices): per-device VMM allocations bound to one multicast object; the pools alias them, and this is
  // declared before the pools so that it outlives them
  std::unique_ptr<kk::NvlsPools> nvls;
  std::vector<kk::Pool> pools;  // per local device
  // What kk_export hands out is fixed once the pools exist: the manifest text and the pool's CUDA IPC handle are built on first use and kept.  Every
  // cell that mounts the model exports again, and the calls underneath (cudaIpcGetMemHandle, cudaGetDeviceProperties) go through the driver's
  // system-wide lock, where they wait behind whatever another process on the host is doing in the driver.
  std::mutex export_mu;
  std::vector<std::string> manifest_cache;               // per local device, empty = not built yet
  std::vector<std::vector<uint8_t>> pool_handle_cache;   // per local device, empty = not asked yet
  std::vector<kk::DevBuf> d_segs;    // per local device: device copy of its part's segment table
  kk::PeerBuf peer[kk::kPeerKinds][KK_MAX_DEVICES];  // [kind][rank]
  // Per local device.  KK_FANOUT_RAW: the raw image (the resident image too), allocated with the pools; empty once released.  Otherwise the
  // resident image (kernel-stage measurement), staged by kk_stage_resident.
  std::vector<kk::DeviceImage> images;
  std::vector<std::vector<uint64_t>> img_off;   // [part][chunk] offset of the chunk buffer inside the raw image
  std::vector<uint32_t> chunk_base;             // prefix sum of chunk counts per part
  // KK_FANOUT_PULL (one process per GPU): this rank's part of the pool, [slice_lo, slice_hi), also lives in slice_buf (a separate,
  // small allocation — the only thing peers have to map); slice_buf[0] corresponds to pool offset slice_base
  kk::DevBuf slice_buf;
  uint64_t slice_base = 0;
  std::vector<std::pair<uint64_t, uint64_t>> part_range;  // [lo, hi) pool bytes every part produces
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
int model_local_device(kk_model* m, int ordinal);  // local device index (into ctx->devs) or throws
std::string model_manifest(kk_model* m, int local);
void model_pool_ipc_handle(kk_model* m, int local, void* handle_64B);  // cudaIpcGetMemHandle of the pool, once per model and device
std::string model_stats(kk_model* m);
void model_stage_resident(kk_model* m);
void model_unstage_resident(kk_model* m);
void model_convert_resident(kk_model* m, float* ms_total, float* ms_per_launch, size_t cap, size_t* n_launches);

}  // namespace kk
